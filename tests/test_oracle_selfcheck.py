"""Self-checks that strengthen the (unpinned) oracle: SURVEY.md §8c."""
import numpy as np
import pytest

from strolle_b200 import scenes
from tests.util import assert_bits_equal, check_within, random_rays, rel_l2


@pytest.fixture(scope="module")
def cornell_oracle(oracle, blue_noise):
    e = oracle.OracleEngine(blue_noise=blue_noise)
    cam = scenes.apply(e, scenes.cornell(96, 64))
    e.tick()
    return e, cam


def test_bvh_invariants(cornell_oracle):
    e, _ = cornell_oracle
    bvh = e.read_scene("bvh").reshape(-1, 4)
    bits = bvh.view(np.uint32)
    tris = e.read_scene("triangles").reshape(-1, 9, 4)
    assert tris.shape[0] == 32
    seen = []
    def visit(ptr, lo, hi, depth):
        assert depth <= 24
        if bits[ptr, 3] == 0:   # internal: [L.min,0][L.max,right_ptr][R.min,0][R.max,0], left child at ptr+4
            lmin, lmax, rmin, rmax = bvh[ptr, :3], bvh[ptr + 1, :3], bvh[ptr + 2, :3], bvh[ptr + 3, :3]
            visit(ptr + 4, lmin, lmax, depth + 1)
            visit(int(bits[ptr + 1, 3]), rmin, rmax, depth + 1)
        else:
            while True:
                flags, tid = int(bits[ptr, 0]), int(bits[ptr, 1])
                seen.append(tid)
                pos = tris[tid, [0, 3, 6], :3]
                if lo is not None:
                    assert (pos >= lo - 1e-6).all() and (pos <= hi + 1e-6).all()
                assert int(bits[ptr, 3]) == 1
                if not (flags & 1):
                    break
                ptr += 1
    visit(0, None, None, 1)
    assert sorted(seen) == list(range(32)), "every triangle is referenced exactly once"
    assert e.bvh_depth() <= 24


def test_bvh_quirk_multi_triangle_leaves(cornell_oracle):
    # quirk C-7: primitives whose centroids share a bit-identical x never split -> leaves with > 1 entry
    e, _ = cornell_oracle
    bits = e.read_scene("bvh").reshape(-1, 4).view(np.uint32)
    leaves = bits[bits[:, 3] == 1]
    assert (leaves[:, 0] & 1).any()


def test_traversal_matches_brute_force(cornell_oracle):
    e, _ = cornell_oracle
    rays = random_rays(20000, 1, (-1.0, 0.0, -1.0), (1.0, 2.0, 3.0))
    hits = e.trace_closest(rays)
    dist, tri = e.trace_brute(rays)
    bvh_tri = hits[:, 9].copy().view(np.uint32)
    assert_bits_equal(hits[:, 8], dist, "closest distance")
    # triangle ids agree except for exact distance ties (different visiting order)
    differ = bvh_tri != tri
    assert differ.mean() < 1e-3
    # any-hit == closest-hit within len
    rays_len = rays.copy()
    rays_len[:, 3] = np.float32(2.0)
    occ = e.trace_any(rays_len)
    assert ((dist < 2.0) == (occ == 1)).all()


def test_deterministic_and_frame_progress(oracle, blue_noise):
    outs = []
    for _ in range(2):
        e = oracle.OracleEngine(blue_noise=blue_noise)
        cam = scenes.apply(e, scenes.cornell(64, 48))
        for _f in range(3):
            e.tick()
            e.render_camera(cam)
        outs.append(e.read_buffer(cam, "output"))
    assert_bits_equal(outs[0], outs[1], "oracle is deterministic")
    assert np.isfinite(outs[0]).all()


def test_libm_variant_agrees_within_tolerance(oracle, blue_noise):
    """Swapping the Cephes-style elementary functions for the host libm moves the image by far less
    than the 1e-3 relative-L2 parity tolerance of BASELINE.json's north_star."""
    imgs = []
    for libm in (False, True):
        e = oracle.OracleEngine(libm=libm, blue_noise=blue_noise)
        cam = scenes.apply(e, scenes.cornell(96, 64))
        e.tick()
        e.render_camera(cam)
        imgs.append(e.read_buffer(cam, "output").reshape(-1, 4)[:, :3])
    assert rel_l2(imgs[0], imgs[1]) < 1e-3
    for op, a, b in [("sin", np.linspace(-7, 7, 1001), None), ("cos", np.linspace(-7, 7, 1001), None), ("acos", np.linspace(-1, 1, 1001), None),
                     ("exp", np.linspace(-20, 20, 1001), None), ("pow", np.linspace(0.001, 1.0, 1001), np.full(1001, 2.2)),
                     ("atan2", np.sin(np.linspace(-3, 3, 1001)), np.cos(np.linspace(-3, 3, 1001)))]:
        x = oracle.math(op, a, b)
        y = oracle.math(op, a, b, libm=True)
        np.testing.assert_allclose(x, y, rtol=2e-6, atol=2e-7)


def test_reference_mode_energy_matches_restir(oracle, blue_noise):
    """Statistical cross-check (SURVEY §8c): the path-traced reference mode and the ReSTIR+SVGF
    image agree in mean radiance on Cornell."""
    e1 = oracle.OracleEngine(blue_noise=blue_noise)
    c1 = scenes.apply(e1, scenes.cornell(96, 54))
    for _ in range(12):
        e1.tick(); e1.render_camera(c1)
    e2 = oracle.OracleEngine(blue_noise=blue_noise)
    c2 = scenes.apply(e2, scenes.cornell(96, 54, mode=scenes.MODE_REFERENCE, ref_depth=2))
    for _ in range(48):
        e2.tick(); e2.render_camera(c2)
    a = e1.read_buffer(c1, "output").reshape(-1, 4)[:, :3].mean()
    b = e2.read_buffer(c2, "output").reshape(-1, 4)[:, :3].mean()
    assert abs(a - b) / b < 0.2


def test_light_slot_protocol(oracle, blue_noise):
    # strolle/src/lights.rs:101-162: removing a light kills its slot for one frame and remaps the tail
    e = oracle.OracleEngine(blue_noise=blue_noise)
    sc = scenes.cornell(32, 32)
    cam = scenes.apply(e, sc)
    e.insert_light(401, scenes.LIGHT_POINT, scenes.point_light((0.5, 1.0, 0.0), 0.1, (1, 1, 1), 10.0))
    e.insert_light(402, scenes.LIGHT_POINT, scenes.point_light((-0.5, 1.0, 0.0), 0.1, (2, 2, 2), 10.0))
    e.tick()
    l0 = e.read_scene("lights").reshape(-1, 28)
    assert e.read_scene("world").view(np.uint32)[0] == 4
    assert (l0[1:4, 16:28] == 0).all(), "created lights upload with zero prev_d* on their first frame"
    e.remove_light(401)
    e.tick()
    l1 = e.read_scene("lights").reshape(-1, 28)
    slot = l1[:, 12].copy().view(np.uint32)
    assert e.read_scene("world").view(np.uint32)[0] == 3
    assert slot[2] == 0xCAFEBABE or slot[3] == 3, "killed / remapped slot markers are visible for one frame"
    e.tick()
    l2 = e.read_scene("lights").reshape(-1, 28)
    assert (l2[:, 12].view(np.uint32) == 0).all()


def test_textured_scene_oracle(oracle, blue_noise):
    """The atlas path of the oracle: textures change the image, the alpha cutout lets light through."""
    sc = scenes.textured_room(96, 54)
    e = oracle.OracleEngine(blue_noise=blue_noise)
    cam = scenes.apply(e, sc)
    for _ in range(3):
        e.tick(); e.render_camera(cam)
    img = e.read_buffer(cam, "output").reshape(54, 96, 4)[..., :3]
    assert np.isfinite(img).all() and img.mean() > 0.01
    mats = e.read_scene("materials").reshape(-1, 28)
    assert mats[0, 4:8].tolist() == [0.0, 0.0, 64 / 8192, 64 / 8192]   # first image sits at the atlas origin
    assert mats[2, 4] == 64 / 8192                                       # second image packed to its right on the shelf
    plain = dict(sc); plain["material_textures"] = {}
    e2 = oracle.OracleEngine(blue_noise=blue_noise)
    c2 = scenes.apply(e2, plain)
    for _ in range(3):
        e2.tick(); e2.render_camera(c2)
    img2 = e2.read_buffer(c2, "output").reshape(54, 96, 4)[..., :3]
    assert rel_l2(img, img2) > 0.05


def test_glam_acos_approx_and_spot_cone(oracle, blue_noise):
    """glam's `acos_approx` (what `Vec3::angle_between` evaluates for the spot-light cone, strolle-gpu/src/light.rs:149-152):
    known answers of the published polynomial (DirectXMath XMScalarACos: exact at +-1, <= 1e-4 rad everywhere, pi-mirrored) and a
    spot light actually cutting its cone in a rendered frame."""
    x = np.concatenate([np.linspace(-1, 1, 20001), [1.5, -1.5]]).astype(np.float32)
    got = oracle.math("acos_approx", x)
    want = np.arccos(np.clip(x.astype(np.float64), -1, 1))
    assert np.abs(got - want).max() < 1e-4
    assert got[20000] == 0.0 and got[0] == np.float32(np.pi)                 # acos_approx(1) = 0, acos_approx(-1) = pi - 0
    assert got[-2] == 0.0 and got[-1] == np.float32(np.pi)                   # out-of-range arguments clamp through max(1 - |x|, 0)
    assert abs(float(got[10000]) - 1.5707963050) < 1e-7                       # the polynomial's constant term at x = 0
    assert np.all(np.diff(got[:20001]) <= 0)                                   # monotone
    # a downward spot above the Cornell floor: lit inside the cone, dark outside, unlike the point light it replaces
    from strolle_b200 import scenes
    lit = {}
    for kind in ("point", "spot"):
        scene = scenes.cornell(64, 48)
        h, _, p = scene["lights"][0]
        if kind == "spot":
            scene["lights"][0] = (h, scenes.LIGHT_SPOT, scenes.spot_light(p[0:3], p[3], p[4:7], p[7], (0.0, -1.0, 0.0), 0.35))
        eo = oracle.OracleEngine(blue_noise=blue_noise)
        co = scenes.apply(eo, scene)
        for _ in range(3):
            eo.tick(); eo.render_camera(co)
        lit[kind] = eo.read_buffer(co, "di_diff_samples").reshape(48, 64, 4)[..., :3].sum(axis=2)
    assert np.isfinite(lit["spot"]).all() and lit["spot"].max() > 0
    assert (lit["spot"] > 0).sum() < 0.7 * (lit["point"] > 0).sum(), "the cone leaves most of the box unlit"


def test_primary_visibility_matches_textbook_float64(oracle, blue_noise):
    """Independent of the reference's code: a float64 pinhole camera (pixel centres through the inverse of the infinite reverse-Z
    projection) and a textbook Möller–Trumbore test over ALL triangles reproduce the oracle's primary pass — the same triangle under
    (nearly) every pixel, and the surface map's depth = distance from the near-plane point along the pixel's ray to the hit."""
    W, H = 96, 64
    sc = scenes.cornell(W, H)
    e = oracle.OracleEngine(blue_noise=blue_noise)
    cam = scenes.apply(e, sc)
    e.tick(); e.render_camera(cam)
    tid = e.read_buffer(cam, "prim_triangle_ids").reshape(H, W, 4)[..., 0].copy().view(np.uint32)
    surface = e.read_buffer(cam, "prim_surface_map_b").reshape(H, W, 4)                # frame 1 writes the "b" half
    depth = surface[..., 2]
    tris = e.read_scene("triangles").reshape(-1, 9, 4).astype(np.float64)               # positions in vec4 0, 3, 6 (triangle.rs:8-21)
    P = sc["camera"]["projection"].reshape(4, 4).astype(np.float64)                     # [column][row]
    T = sc["camera"]["transform"].reshape(4, 4).astype(np.float64)
    origin, R, near = T[3, :3], T[:3, :3], 0.1
    ys, xs = np.mgrid[0:H, 0:W]
    dv = np.stack([((xs + 0.5) / W * 2 - 1) / P[0, 0], (1 - (ys + 0.5) / H * 2) / P[1, 1], -np.ones((H, W))], -1)
    dw = dv[..., 0:1] * R[0] + dv[..., 1:2] * R[1] + dv[..., 2:3] * R[2]
    dw /= np.linalg.norm(dw, axis=-1, keepdims=True)
    best = np.full((H, W), np.inf); who = np.full((H, W), 0xFFFFFFFF, dtype=np.uint32)
    normal = np.zeros((H, W, 3))
    for i, t3 in enumerate(tris):
        p0, e1, e2 = t3[0, :3], t3[3, :3] - t3[0, :3], t3[6, :3] - t3[0, :3]
        pv = np.cross(dw, e2); det = (pv * e1).sum(-1)
        with np.errstate(divide="ignore", invalid="ignore"):
            inv = 1.0 / det
            tv = origin - p0
            u = (pv * tv).sum(-1) * inv
            qv = np.cross(tv, e1)
            v = (dw * qv).sum(-1) * inv
            t = (qv * e2).sum(-1) * inv
        ok = (np.abs(det) > 1e-12) & (u >= 0) & (v >= 0) & (u + v <= 1) & (t > 1e-9) & (t < best)
        best = np.where(ok, t, best); who = np.where(ok, np.uint32(i), who)
        with np.errstate(invalid="ignore"):
            n = t3[4, :3] * u[..., None] + t3[7, :3] * v[..., None] + t3[1, :3] * (1 - u - v)[..., None]    # vertex normals in vec4 1, 4, 7
            n = n / np.linalg.norm(n, axis=-1, keepdims=True) * np.sign(det)[..., None]                    # two-sided: faces the ray
        normal = np.where(ok[..., None], n, normal)
    same = who == tid
    assert same.mean() > 0.995, f"triangle under the pixel: {same.mean():.4f} agree"      # the rest sit on shared edges
    assert ((tid == 0xFFFFFFFF) == np.isinf(best))[same].all()
    hit = same & (tid != 0xFFFFFFFF)
    cos = -dv[..., 2] / np.linalg.norm(dv, axis=-1)
    err = np.abs(depth[hit] - (best[hit] - near / cos[hit]))
    assert err.max() < 2e-5, err.max()
    # the surface map's normal: standard octahedral decode of its first two components == the interpolated vertex normal
    m = surface[..., 0:2].astype(np.float64) * 2 - 1
    dec = np.stack([m[..., 0], m[..., 1], 1 - np.abs(m[..., 0]) - np.abs(m[..., 1])], -1)
    fold = np.maximum(-dec[..., 2], 0)
    dec[..., 0] -= np.copysign(fold, dec[..., 0]); dec[..., 1] -= np.copysign(fold, dec[..., 1])
    dec /= np.linalg.norm(dec, axis=-1, keepdims=True)
    assert np.abs(dec[hit] - normal[hit]).max() < 1e-5


def test_ray_stream_matches_float64_brute_force(cornell_oracle):
    """Ray::trace on random rays against a float64 Möller–Trumbore over all triangles (written from the textbook definition, two-sided,
    no BVH): same closest triangle except at distance ties, hit distance within f32 rounding of the f64 one."""
    e, _ = cornell_oracle
    rays = random_rays(6000, 3, (-1.0, 0.0, -1.0), (1.0, 2.0, 3.0))
    hits = e.trace_closest(rays)
    tris = e.read_scene("triangles").reshape(-1, 9, 4).astype(np.float64)
    o, d = rays[:, 0:3].astype(np.float64), rays[:, 4:7].astype(np.float64)
    best = np.full(len(rays), np.inf); who = np.full(len(rays), 0xFFFFFFFF, dtype=np.uint32)
    for i, t3 in enumerate(tris):
        p0, e1, e2 = t3[0, :3], t3[3, :3] - t3[0, :3], t3[6, :3] - t3[0, :3]
        pv = np.cross(d, e2); det = pv @ e1
        with np.errstate(divide="ignore", invalid="ignore"):
            inv = 1.0 / det
            tv = o - p0
            u = (pv * tv).sum(-1) * inv
            qv = np.cross(tv, e1)
            v = (d * qv).sum(-1) * inv
            t = (qv @ e2) * inv
        ok = (np.abs(det) > 1e-12) & (u >= 0) & (v >= 0) & (u + v <= 1) & (t > 1e-9) & (t < best)
        best = np.where(ok, t, best); who = np.where(ok, np.uint32(i), who)
    got_tri = hits[:, 9].copy().view(np.uint32)
    got_t = hits[:, 8].astype(np.float64)
    miss = np.isinf(best)
    assert ((got_tri == 0xFFFFFFFF) == miss).mean() > 0.999
    both = ~miss & (got_tri != 0xFFFFFFFF)
    assert (got_tri[both] == who[both]).mean() > 0.995
    same = both & (got_tri == who)
    assert (np.abs(got_t[same] - best[same]) <= 4e-6 * np.maximum(1.0, best[same])).all()


def test_ref64_constants(oracle):
    """The Cephes error constants tests/ref64_svgf.py and tests/ref64_restir.py build their strict bounds on, measured through
    oracle.math (bit-identical to the device functions, test_device_math_bit_exact)."""
    from tests import ref64_svgf as R
    x = np.linspace(-87.0, 0.0, 400001).astype(np.float32)
    t = np.exp(x.astype(np.float64))
    assert (np.abs(oracle.math("exp", x) - t) / t).max() <= R.EXP_REL
    b = (np.arange(256) / np.float32(255.0)).astype(np.float32)[1:]
    t = b.astype(np.float64) ** 2.2
    assert (np.abs(oracle.math("pow", b, np.full_like(b, 2.2)) - t) / t).max() <= R.POW22_REL
    x = np.linspace(0.0031308, 1.0, 400001).astype(np.float32)
    p = np.float32(1.0) / np.float32(2.4)
    t = x.astype(np.float64) ** float(p)
    assert (np.abs(oracle.math("pow", x, np.full_like(x, p)) - t) / t).max() <= R.POW_INV24_REL
    # the strict sin / cos on the angles 2 pi r, r in [0, 1), that the ReSTIR disk and sphere samples take (tests/ref64_restir.py)
    from tests import ref64_restir as Q
    x = np.concatenate([np.linspace(0.0, 2 * np.pi, 400001), np.random.RandomState(1).uniform(0, 2 * np.pi, 10 ** 6)]).astype(np.float32)
    for op, fn in (("sin", np.sin), ("cos", np.cos)):
        assert np.abs(oracle.math(op, x) - fn(x.astype(np.float64))).max() <= Q.SIN_ABS, op
    # the strict acos and atan2 that Atmosphere::sample's zenith angle, horizon and azimuth take, on all of [-1, 1] (densely toward
    # +-1) and on points of every angle at radii 1e-3 to 1.26
    rng = np.random.RandomState(2)
    x = np.concatenate([np.linspace(-1.0, 1.0, 400001), 1 - np.logspace(-8, 0, 10 ** 5), np.logspace(-8, 0, 10 ** 5) - 1]).astype(np.float32)
    x = x[np.abs(x) <= 1]
    assert np.abs(oracle.math("acos", x) - np.arccos(x.astype(np.float64))).max() <= Q.ACOS_ABS
    a, r = rng.uniform(0, 2 * np.pi, 10 ** 6), 10 ** rng.uniform(-3, 0.1, 10 ** 6)
    ys, xs = (r * np.sin(a)).astype(np.float32), (r * np.cos(a)).astype(np.float32)
    assert np.abs(oracle.math("atan2", ys, xs) - np.arctan2(ys.astype(np.float64), xs.astype(np.float64))).max() <= Q.ATAN2_ABS


def _svgf_chain_check(oracle, blue_noise, scene, frames=6, moves=(3, 4, 5)):
    """The f64 chain of tests/ref64_svgf.py against the strict oracle, stage by stage.  From the buffers at the end of frame f - 1
    (history) and of frame f (this frame's samples, surface, reprojection, G-buffer), K20 must give `moments[cur]`, K20 -> K21 ->
    iteration 0 `prev_colors`, -> iterations 1-3 `stash`, -> iteration 4 `curr_colors`, and composition `output`, every value within
    the strict-tier bound.  Returns the largest error / bound per stage."""
    from tests import ref64_svgf as R
    e = oracle.OracleEngine(blue_noise=blue_noise)
    cam = scenes.apply(e, scene)
    c = scene["camera"]
    w, h = c["w"], c["h"]
    rd = lambda n: e.read_buffer(cam, n).reshape(h, w, 4)
    ratios = {}
    prev = None
    for f in range(1, frames + 1):
        if f in moves:
            t = np.asarray(c["transform"], dtype=np.float32).copy().reshape(16)     # column-major: translation in 12-14
            t[12] += np.float32(0.011 * f); t[13] += np.float32(0.005 * f)
            e.update_camera(cam, c["mode"], c["denoise"], c["ref_depth"], w, h, t, c["projection"])
        e.tick(); e.render_camera(cam)
        cur = "b" if f % 2 == 1 else "a"
        now = {n: rd(n) for n in ("di_diff_samples", "gi_diff_samples", "reprojection_map", f"prim_surface_map_{cur}", f"prim_gbuffer_d0_{cur}",
                                  f"prim_gbuffer_d1_{cur}", "di_spec_samples", "gi_spec_samples", "ref_colors", "output",
                                  "di_diff_moments_a", "di_diff_moments_b", "gi_diff_moments_a", "gi_diff_moments_b",
                                  "di_diff_prev_colors", "gi_diff_prev_colors", "di_diff_stash", "gi_diff_stash",
                                  "di_diff_curr_colors", "gi_diff_curr_colors")}
        if prev is None:
            prev = {k: np.zeros_like(v) for k, v in now.items()}
        old = "a" if cur == "b" else "b"
        sm = now[f"prim_surface_map_{cur}"]
        k20, k20b = {}, {}
        for sig in ("di", "gi"):
            r = R.reproject(now[f"{sig}_diff_samples"], sm, now["reprojection_map"], prev[f"{sig}_diff_prev_colors"], prev[f"{sig}_diff_moments_{old}"])
            mom_want = np.where(r["sky"][..., None], prev[f"{sig}_diff_moments_{cur}"], r["moment"])
            ratios["K20"] = max(ratios.get("K20", 0), check_within(now[f"{sig}_diff_moments_{cur}"], mom_want, r["b_moment"], f"{scene.get('name')} f{f} K20 {sig} moments"))
            k20[sig], k20b[sig] = r["color"], r["b_color"]
        moms = {s: now[f"{s}_diff_moments_{cur}"] for s in ("di", "gi")}
        v = R.estimate_variance(sm, k20, moms, d_colors=k20b)
        di, gi, bdi, bgi = v["di"], v["gi"], v["b_di"], v["b_gi"]
        sky = v["sky"][..., None]
        targets = {0: "prev_colors", 3: "stash", 4: "curr_colors"}
        for it in range(5):
            r = R.wavelet(sm, di, gi, it, f, blue_noise, bdi, bgi)
            di, bdi, bgi = r["di"], r["b_di"], r["b_gi"]
            gi = np.where(sky, 0.0, r["gi"])
            if it in targets:
                for sig, want, b in (("di", di, bdi), ("gi", gi, bgi)):
                    got = now[f"{sig}_diff_{targets[it]}"]
                    if sig == "gi":
                        got = np.where(sky, 0.0, got)
                    key = f"K22 iteration {it}"
                    ratios[key] = max(ratios.get(key, 0), check_within(got, want, b, f"{scene.get('name')} f{f} {key} {sig}"))
        col, b = R.compose(0, now[f"prim_gbuffer_d0_{cur}"], now[f"prim_gbuffer_d1_{cur}"], di, gi, now["di_spec_samples"], now["gi_spec_samples"],
                           now["ref_colors"], bdi, bgi)
        ratios["composition"] = max(ratios.get("composition", 0), check_within(now["output"][..., :3], col, b, f"{scene.get('name')} f{f} output"))
        assert (now["output"][..., 3] == 1).all()
        prev = now
    return ratios


@pytest.mark.parametrize("which", ["cornell", "demo_level"])
def test_svgf_float64_chain_matches_oracle(oracle, blue_noise, which):
    """tests/ref64_svgf.py against the strict oracle on Cornell 96x64 over 18 frames and a small dungeon over 6 (camera moving on
    frames 3-5, so K20's bilinear path runs; the history crosses 4 and, on Cornell, reaches its cap of 16): the restatement reads the reference the way the oracle does, and its
    strict-tier bound holds.  The bound must not be vacuous: the oracle's rounding uses a visible part of it somewhere."""
    scene = scenes.cornell(96, 64) if which == "cornell" else scenes.demo_level(80, 45)
    scene.setdefault("name", which)
    ratios = _svgf_chain_check(oracle, blue_noise, scene, frames=18 if which == "cornell" else 6)   # 18: the history reaches its cap of 16
    assert max(ratios.values()) > 1e-3, ratios


def test_transmittance_lut_is_physically_plausible(oracle, blue_noise):
    """The atmosphere's transmittance LUT against closed-form physics with the published constants of the model the reference implements
    (Hillaire 2020: Rayleigh 5.802 / 13.558 / 33.1 e-6 per m with an 8 km scale height, Mie extinction 8.396e-6 with 1.2 km, ozone
    0.650 / 1.881 / 0.085 e-6 over a 30 km tent): looking straight up from the ground the optical depth is sum(beta_i * column_i).
    The LUT is a fixed-step numerical integral, so the match is loose (5 %); it also has to be 1 at the top of the atmosphere, 0 below
    the horizon at ground level, and grow with the elevation of the view direction."""
    e = oracle.OracleEngine(blue_noise=blue_noise)
    cam = scenes.apply(e, scenes.demo_level(64, 36))
    e.tick(); e.render_camera(cam)
    t = e.read_scene("transmittance_lut").reshape(64, 256, 4)[..., :3].astype(np.float64)   # [height][cos zenith -1..1]
    tau = np.array([5.802, 13.558, 33.1]) * 1e-6 * 8000.0 + 8.396e-6 * 1200.0 + np.array([0.650, 1.881, 0.085]) * 1e-6 * 15000.0
    assert np.abs(t[0, 255] - np.exp(-tau)).max() < 0.05, (t[0, 255], np.exp(-tau))
    assert (t[63, 128:] > 0.999).all() and (t[0, :100] == 0).all()
    assert (np.diff(t[0, 128:], axis=0) >= -2e-3).all(), "transmittance grows towards the zenith"
    assert (t >= 0).all() and (t <= 1).all()


def _restir_chain_check(oracle, blue_noise, scene, frames=13, moves=(3, 5, 8, 11), edge_lights=False, extra_lights=0, remove=9001):
    """K5 (DI sampling), K6 (DI temporal resampling), K7 (the spatial tap choice), K8 (the spatial visibility rays), K9 (DI spatial
    merge, and K7 + K8 + K9 composed as the fused launch is checked) and K10 (DI resolving) of the strict
    oracle against tests/ref64_restir.py, pass by pass: the frame is stepped with render_range, each pass's inputs are read right
    before it runs and its outputs right after.  `extra_lights` small point lights are added before the first frame; `remove` is
    the light taken out on frame 10 (9001, the last one, kills its slot; one from the middle of the list remaps the last slot)."""
    from tests import ref64_restir as Q
    c = scene["camera"]
    w, h = c["w"], c["h"]
    e = oracle.OracleEngine(blue_noise=blue_noise)
    cam = scenes.apply(e, scene)
    t = np.asarray(c["transform"], np.float32).reshape(16).copy()
    t_prev = t.copy()          # the camera before the last update_camera: what the engine keeps as the previous camera
    stats = {"K6": [0.0, {}, 0], "K6 tight": {k: [0, 0] for k in ("m", "w", "pdf")}, "K6 branches": [0, 0, 0], "K8": [0, 0],
             "K9": [0.0, 0, 0], "K10": [0.0, 0], "K9 tight": [0, 0], "K5": [0.0, {}, 0, 0],
             "K5 tight": {k: [0, 0] for k in ("w", "light_point")}, "K7": [0.0, 0, 0], "K7 tight": [0, 0], "K7 branches": {}}
    if edge_lights:
        from tests.test_restir_reference import edge_lights as add_lights
        add_lights(e)
    from tests.test_restir_reference import many_lights
    many_lights(e, extra_lights)
    for f in range(1, frames + 1):
        if f in moves:
            t_prev = t.copy()
            t[12] += np.float32(0.013 * f); t[13] += np.float32(0.004 * f)
            e.update_camera(cam, c["mode"], c["denoise"], c["ref_depth"], w, h, t, c["projection"])
        if f == 4:
            e.insert_light(9001, scenes.LIGHT_POINT, scenes.point_light((0.2, 1.0, 0.3), 0.08, (3.0, 2.0, 1.0), 6.0))
        if f == 7:
            e.insert_light(9001, scenes.LIGHT_POINT, scenes.point_light((-0.3, 0.8, 0.1), 0.08, (3.0, 2.0, 1.0), 6.0))
        if f == 10:
            e.remove_light(remove)
        e.tick()
        sched = e.frame_schedule(cam)
        k5, k6, k7, k8, k9, k10 = (sched.index(p) for p in (1, 2, 3, 4, 5, 6))
        rd = lambda n: e.read_buffer(cam, n)
        cur = "b" if f % 2 == 1 else "a"
        old = "a" if cur == "b" else "b"
        e.render_range(cam, 0, k5 - 1)
        r1 = rd("di_reservoirs_1")
        k5r = Q.di_sampling(Q.ndc_to_world(t, c["projection"]), w, h, rd(f"prim_gbuffer_d0_{cur}").reshape(h, w, 4),
                            rd(f"prim_gbuffer_d1_{cur}").reshape(h, w, 4), e.read_scene("lights"),
                            e.read_scene("world")[:1].view(np.uint32)[0], blue_noise, Q.dispatch_seed(0xC0FFEE, f, 1), f, fast=False)
        e.render_range(cam, k5, k5)
        s5 = Q.check_sampling(rd("di_reservoirs_1"), r1, k5r, lambda x: oracle.math("sin", x), lambda x: oracle.math("cos", x),
                              e.trace_any, f"f{f} K5")
        assert s5["disagree"] == 0, f"f{f} K5: {s5['disagree']} of {s5['traced']} occluded bits differ from trace_any"
        assert_bits_equal(s5["got"][:, 4:7], s5["lp_f32"], f"f{f} K5 light point against its strict f32 rebuild")
        k5s = stats["K5"]
        stats["K5"] = [max(k5s[0], s5["ratio"]), {k: k5s[1].get(k, 0) + v for k, v in s5["undecided"].items()}, k5s[2] + s5["n"],
                       k5s[3] + s5["traced"]]
        for k, (tt, nn) in s5["tight"].items():
            stats["K5 tight"][k][0] += tt; stats["K5 tight"][k][1] += nn
        e.render_range(cam, k5 + 1, k6 - 1)
        gb = [rd(f"prim_gbuffer_d{k}_{cur}").reshape(h, w, 4) for k in (0, 1)]
        gb_prev = [rd(f"prim_gbuffer_d{k}_{old}").reshape(h, w, 4) for k in (0, 1)]
        r1, r0 = rd("di_reservoirs_1"), rd("di_reservoirs_0")
        k6r = Q.di_temporal(Q.ndc_to_world(t, c["projection"]), Q.ndc_to_world(t_prev, c["projection"]), w, h, gb, gb_prev,
                            rd("reprojection_map"), e.read_scene("lights"), r1, r0, Q.dispatch_seed(0xC0FFEE, f, 2), fast=False)
        e.render_range(cam, k6, k6)
        ratio, und, npx, _ = Q.check_temporal(rd("di_reservoirs_1"), r1, k6r, f"f{f} K6")
        # the composition the fused K5 + K6 launch is checked against: K5's restated sample (bounded w and light point, the
        # occluded bit from trace_any of the strict f32 rebuild) handed to K6's restatement; on the strict oracle every pixel matches
        lhs = Q.sampling_lhs(k5r, lambda x: oracle.math("sin", x), lambda x: oracle.math("cos", x), e.trace_any)
        kc6 = Q.di_temporal(Q.ndc_to_world(t, c["projection"]), Q.ndc_to_world(t_prev, c["projection"]), w, h, gb, gb_prev,
                            rd("reprojection_map"), e.read_scene("lights"), None, r0, Q.dispatch_seed(0xC0FFEE, f, 2), fast=False, lhs=lhs)
        Q.check_temporal(rd("di_reservoirs_1"), r1, kc6, f"f{f} K5-K6 composed")
        s = stats["K6"]
        stats["K6"] = [max(s[0], ratio), {k: s[1].get(k, 0) + v for k, v in und.items()}, s[2] + npx]
        for k, (tt, nn) in Q.temporal_tight(k6r).items():
            stats["K6 tight"][k][0] += tt; stats["K6 tight"][k][1] += nn
        stats["K6 branches"] = [a + k6r[b] for a, b in zip(stats["K6 branches"], ("reprojected", "killed", "remapped"))]
        e.render_range(cam, k6 + 1, k7 - 1)
        p0, p1, r1 = rd("di_diff_samples"), rd("di_diff_curr_colors"), rd("di_reservoirs_1")
        k7r = Q.di_spatial_pick(Q.ndc_to_world(t, c["projection"]), w, h, rd(f"prim_gbuffer_d0_{cur}"), rd(f"prim_gbuffer_d1_{cur}"),
                                e.read_scene("lights"), r1, Q.dispatch_seed(0xC0FFEE, f, 3), f, fast=False)
        e.render_range(cam, k7, k7)
        s7 = Q.check_spatial_pick(rd("di_diff_samples"), rd("di_diff_curr_colors"), p0, p1, k7r, f"f{f} K7")
        stats["K7"] = [max(stats["K7"][0], s7["ratio"]), stats["K7"][1] + s7["undecided"], stats["K7"][2] + s7["pairs"]]
        stats["K7 tight"] = [a + b for a, b in zip(stats["K7 tight"], s7["tight"])]
        stats["K7 branches"] = {k: stats["K7 branches"].get(k, 0) + v for k, v in k7r["branches"].items()}
        e.render_range(cam, k7 + 1, k8 - 1)
        b0, b1 = rd("di_diff_samples"), rd("di_diff_curr_colors")
        e.render_range(cam, k8, k8)
        traced, bad = Q.check_spatial_trace(b0, b1, rd("di_diff_stash"), e.trace_any, f"f{f} K8")
        assert bad == 0, f"f{f} K8: {bad} of {traced} visibility bits differ from trace_any"
        stats["K8"] = [stats["K8"][0] + traced, stats["K8"][1] + bad]
        e.render_range(cam, k8 + 1, k9 - 1)
        r1, stash = rd("di_reservoirs_1"), rd("di_diff_stash")
        e.render_range(cam, k9, k9)
        r2 = rd("di_reservoirs_2")
        k9r = Q.di_spatial_sample(r1, stash, Q.dispatch_seed(0xC0FFEE, f, 5), f, w, h, fast=False)
        ratio, und, merged, _ = Q.check_spatial_sample(r2, r1, k9r, f"f{f} K9")
        # the composition the fused K7 + K8 + K9 launch is checked against: K7's restatement, trace_any of its rays rebuilt in strict
        # f32, K9's restatement with bounded pdfs; on the strict oracle every pair must match with each visibility bit as traced
        kc = Q.di_spatial_sample(r1, Q.pick_stash(k7r, e.trace_any), Q.dispatch_seed(0xC0FFEE, f, 5), f, w, h, fast=False)
        Q.check_spatial_sample(r2, r1, kc, f"f{f} K7-K9 composed")
        stats["K9"] = [max(stats["K9"][0], ratio), stats["K9"][1] + und, stats["K9"][2] + merged]
        frac, n = Q.spatial_sample_tight(k9r)
        stats["K9 tight"] = [stats["K9 tight"][0] + round(frac * n), stats["K9 tight"][1] + n]
        e.render_range(cam, k9 + 1, k10 - 1)
        d0, d1 = rd(f"prim_gbuffer_d0_{cur}").reshape(h, w, 4), rd(f"prim_gbuffer_d1_{cur}").reshape(h, w, 4)
        r2 = rd("di_reservoirs_2")
        e.render_range(cam, k10, k10)
        n2w = Q.ndc_to_world(t, c["projection"])
        k10r = Q.di_resolving(n2w, w, h, d0, d1, e.read_scene("lights"), r2, rd("di_reservoirs_0"), fast=False,
                              atm=Q.atmosphere_inputs(e))
        ratio, und, _ = Q.check_resolving(rd("di_diff_samples").reshape(h, w, 4), rd("di_spec_samples").reshape(h, w, 4),
                                          rd("di_reservoirs_0"), k10r, f"f{f} K10", check_within)
        stats["K10"] = [max(stats["K10"][0], ratio), stats["K10"][1] + und]
        e.render_range(cam, k10 + 1, -1)
    return stats


def test_oracle_render_range_is_render_camera(oracle, blue_noise):
    """Stepping a frame pass by pass with render_range leaves every buffer exactly as render_camera does, over frames that cover
    both GI cycles; the step list is the one frame_schedule reports."""
    from tests.util import CAMERA_BUFFERS
    outs = []
    for stepped in (False, True):
        e = oracle.OracleEngine(blue_noise=blue_noise)
        cam = scenes.apply(e, scenes.cornell(40, 28))
        for f in range(1, 8):
            e.tick()
            if stepped:
                sched = e.frame_schedule(cam)
                assert sched[0] == 0 and sched[-1] == 20 and sched.count(19) == 5
                for i in range(len(sched)):
                    e.render_range(cam, i, i)
            else:
                e.render_camera(cam)
        outs.append({n: e.read_buffer(cam, n) for n in CAMERA_BUFFERS})
    for n in CAMERA_BUFFERS:
        assert_bits_equal(outs[0][n], outs[1][n], n)


@pytest.mark.parametrize("which", ["cornell", "demo_level", "cornell_spots", "textured_room", "cornell_edge_lights",
                                   "cornell_many_lights", "cornell_remap"])
def test_restir_float64_chain_matches_oracle(oracle, blue_noise, which):
    """The float64 restatement of K6, K8, K9 and K10 reproduces the strict oracle within its bound over 13 frames (both GI cycles),
    with the camera moving and a light inserted, moved and removed mid-run; the textured room's metallic box exercises the specular
    lobe.  Many lights: 23 in all, so K5 draws 16 of them and K6 resamples among lights that are not the first few.  Remap: a light
    is removed from the middle of the list, so K6 sees a remapped slot as well as the killed one.  The oracle and the CUDA kernels
    were written from one reading of the reference; this checks that reading against an independent one without a GPU."""
    scene = {"cornell": lambda: scenes.cornell(96, 64), "demo_level": lambda: scenes.demo_level(80, 45),
             "cornell_spots": lambda: scenes.cornell_spots(72, 48), "textured_room": lambda: scenes.textured_room(80, 44),
             "cornell_edge_lights": lambda: scenes.cornell(72, 48), "cornell_many_lights": lambda: scenes.cornell(72, 48),
             "cornell_remap": lambda: scenes.cornell(72, 48)}[which]()
    from tests.test_restir_reference import MANY_LIGHTS, REMAP_REMOVED
    stats = _restir_chain_check(oracle, blue_noise, scene, edge_lights=which == "cornell_edge_lights",
                                extra_lights=MANY_LIGHTS if which in ("cornell_many_lights", "cornell_remap") else 0,
                                remove=REMAP_REMOVED if which == "cornell_remap" else 9001)
    k6, k5 = stats["K6"], stats["K5"]
    print(f"\n{which}: K5 ratio {k5[0]:.3g} over {k5[2]} pixels, undecided {k5[1]}, {k5[3]} shadow rays, tight {stats['K5 tight']}; "
          f"K6 ratio {k6[0]:.3g} over {k6[2]} pixels, undecided {k6[1]}, reprojected / killed / remapped "
          f"{stats['K6 branches']}; K8 {stats['K8'][0]} rays traced, {stats['K8'][1]} differ; K9 ratio {stats['K9'][0]:.3g}, "
          f"undecided {stats['K9'][1]} of {stats['K9'][2]} merges; K10 ratio {stats['K10'][0]:.3g}, undecided specular {stats['K10'][1]}; "
          f"K7 ratio {stats['K7'][0]:.3g}, undecided {stats['K7'][1]} of {stats['K7'][2]} pairs, tight {stats['K7 tight']}, "
          f"branches {stats['K7 branches']}")
    assert stats["K9"][2] > 0 and stats["K9"][1] <= 0.01 * stats["K9"][2]
    assert 1e-3 < stats["K10"][0] <= 1 and 1e-3 < stats["K9"][0] <= 1 and 1e-3 < k6[0] <= 1
    assert stats["K9 tight"][0] >= 0.99 * stats["K9 tight"][1] > 0, stats["K9 tight"]
    from tests import ref64_restir as Q
    from tests.ref64_restir import tight_ok
    assert tight_ok(stats["K6 tight"]), stats["K6 tight"]
    assert all(v <= 0.01 * k6[2] for v in k6[1].values()), k6[1]
    assert stats["K6 branches"][0] > 0 and stats["K8"][0] > 0
    assert 1e-3 < k5[0] <= 1 and k5[3] > 0 and Q.sampling_tight_ok(stats["K5 tight"]), stats["K5 tight"]
    assert all(v <= 0.01 * k5[2] for v in k5[1].values()), k5[1]
    k7 = stats["K7"]
    assert 1e-3 < k7[0] <= 1 and k7[1] <= 0.01 * k7[2] and Q.pick_tight_ok(stats["K7 tight"]), (k7, stats["K7 tight"])
    if which.startswith("cornell"):     # a reprojected reservoir named light 9001 (or the light removed) after its removal
        assert stats["K6 branches"][1] > 0
    if which == "cornell_remap":
        assert stats["K6 branches"][2] > 0, "no reprojected reservoir named the remapped slot"
