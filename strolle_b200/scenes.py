"""Scene descriptions (input data) for the benchmark configurations.

A scene is plain data: meshes, materials, instances, lights, sun, camera — the
arguments a host application would pass through the Engine API
(strolle/src/lib.rs:161-245).  `apply(engine, scene)` drives any object exposing
that API (the CUDA engine in strolle_b200.engine, or the test oracle).
"""
import json
import math
import os

import numpy as np

_ASSETS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "assets")

MODE_IMAGE, MODE_DI_DIFFUSE, MODE_DI_SPECULAR, MODE_GI_DIFFUSE, MODE_GI_SPECULAR, MODE_BVH_HEATMAP, MODE_REFERENCE = range(7)
LIGHT_POINT, LIGHT_SPOT = 1, 2


def blue_noise():
    """256x256 RGBA8 blue-noise tile (strolle/assets/blue-noise.png as raw bytes)."""
    return np.fromfile(os.path.join(_ASSETS, "blue_noise_256_rgba8.bin"), dtype=np.uint8).reshape(256, 256, 4)


def perspective_infinite_reverse_rh(fov_y, aspect, near):
    """glam Mat4::perspective_infinite_reverse_rh, column-major 16 floats (Bevy's default projection)."""
    f = np.float32(1.0) / np.float32(math.tan(0.5 * fov_y))
    m = np.zeros((4, 4), dtype=np.float32)  # m[col][row]
    m[0][0] = f / np.float32(aspect)
    m[1][1] = f
    m[2][3] = -1.0
    m[3][2] = near
    return m.reshape(-1)


def look_at_transform(eye, target, up=(0.0, 1.0, 0.0)):
    """Bevy Transform::from_translation(eye).looking_at(target, up) as a column-major Mat4."""
    eye = np.asarray(eye, dtype=np.float64)
    fwd = np.asarray(target, dtype=np.float64) - eye
    fwd /= np.linalg.norm(fwd)
    back = -fwd
    right = np.cross(np.asarray(up, dtype=np.float64), back)
    right /= np.linalg.norm(right)
    upv = np.cross(back, right)
    m = np.zeros((4, 4), dtype=np.float32)
    m[0][:3] = right
    m[1][:3] = upv
    m[2][:3] = back
    m[3][:3] = eye
    m[3][3] = 1.0
    return m.reshape(-1)


def material(base_color, emissive=(0, 0, 0, 0), perceptual_roughness=1.0, metallic=0.0, reflectance=0.5, ior=1.0):
    return np.array(list(base_color) + list(emissive) + [perceptual_roughness, metallic, reflectance, ior], dtype=np.float32)


def point_light(position, radius, color, rng):
    return np.array(list(position) + [radius] + list(color) + [rng, 0, 0, 0, 0], dtype=np.float32)


def spot_light(position, radius, color, rng, direction, angle):
    """Light::Spot (strolle/src/light.rs:14-22): a point light restricted to a cone of half-angle `angle` around `direction`."""
    return np.array(list(position) + [radius] + list(color) + [rng] + list(direction) + [angle], dtype=np.float32)


def tri36(positions, normals, uvs=None, tangents=None):
    uvs = uvs if uvs is not None else [[0, 0]] * 3
    tangents = tangents if tangents is not None else [[0, 0, 0, 0]] * 3
    return np.concatenate([np.asarray(positions, np.float32).reshape(-1), np.asarray(normals, np.float32).reshape(-1),
                           np.asarray(uvs, np.float32).reshape(-1), np.asarray(tangents, np.float32).reshape(-1)])


def affine_from_colmajor4x4(m16):
    m = np.asarray(m16, dtype=np.float32).reshape(4, 4)  # m[col][row]
    return np.concatenate([m[0][:3], m[1][:3], m[2][:3], m[3][:3]]).astype(np.float32)


IDENTITY_AFFINE = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0], dtype=np.float32)


def cornell(width=1920, height=1080, mode=MODE_IMAGE, denoise=True, ref_depth=1):
    """Config C1/C2/C4/C5 (BASELINE.md §2.1): Cornell box, 32 triangles, one point light.

    bevy-strolle/examples/cornell.rs:39-94: camera eye (0,1,3.2) -> (0,1,0), point light
    (0,1.5,0.5) r=0.15 range 20 intensity 50, sun altitude -1.
    """
    doc = json.load(open(os.path.join(_ASSETS, "cornell.json")))
    meshes, materials, instances = {}, {}, []
    for i, m in enumerate(doc["materials"]):
        materials[100 + i] = (material(m["base_color"], perceptual_roughness=m["perceptual_roughness"], metallic=m["metallic"]), False)
    for i, m in enumerate(doc["meshes"]):
        tris = np.stack([tri36(t["positions"], t["normals"]) for t in m["triangles"]])
        meshes[200 + i] = tris
        instances.append((300 + i, 200 + i, 100 + m["material"], affine_from_colmajor4x4(m["transform_colmajor"])))
    intensity = 50.0 / (4.0 * math.pi)
    lights = [(400, LIGHT_POINT, point_light((0.0, 1.5, 0.5), 0.15, (intensity,) * 3, 20.0))]
    cam = dict(mode=mode, denoise=denoise, ref_depth=ref_depth, w=width, h=height,
               transform=look_at_transform((0.0, 1.0, 3.2), (0.0, 1.0, 0.0)),
               projection=perspective_infinite_reverse_rh(math.pi / 4.0, width / height, 0.1))
    return dict(name="cornell", meshes=meshes, materials=materials, instances=instances, lights=lights, sun=(0.0, -1.0), camera=cam)


def cornell_spots(width=160, height=120, **kw):
    """Cornell box with two Light::Spot lights next to its point light (a narrow one pointing down, a wide oblique one)."""
    scene = cornell(width, height, **kw)
    h = scene["lights"][0][0]
    scene["lights"].append((h + 1, LIGHT_SPOT, spot_light((0.3, 1.8, 0.2), 0.1, (8.0, 6.0, 4.0), 20.0, (0.0, -1.0, 0.0), 0.35)))
    scene["lights"].append((h + 2, LIGHT_SPOT, spot_light((-0.6, 1.2, 1.5), 0.05, (2.0, 3.0, 5.0), 20.0, (0.4, -0.5, -0.77), 1.1)))
    return scene


def _box(lo, hi):
    lo, hi = np.asarray(lo, np.float32), np.asarray(hi, np.float32)
    c = [np.array([x, y, z], np.float32) for x in (lo[0], hi[0]) for y in (lo[1], hi[1]) for z in (lo[2], hi[2])]
    faces = [((0, 1, 3, 2), (-1, 0, 0)), ((4, 6, 7, 5), (1, 0, 0)), ((0, 4, 5, 1), (0, -1, 0)), ((2, 3, 7, 6), (0, 1, 0)),
             ((0, 2, 6, 4), (0, 0, -1)), ((1, 5, 7, 3), (0, 0, 1))]
    tris = []
    for (a, b, cc, d), n in faces:
        tris.append(tri36([c[a], c[b], c[cc]], [n] * 3, [[0, 0], [1, 0], [1, 1]]))
        tris.append(tri36([c[a], c[cc], c[d]], [n] * 3, [[0, 0], [1, 1], [0, 1]]))
    return tris


def _torus(major=0.5, minor=0.25, nu=24, nv=12):
    tris = []
    def pt(i, j):
        u, v = 2 * math.pi * i / nu, 2 * math.pi * j / nv
        cx, cz = math.cos(u), math.sin(u)
        p = np.array([(major + minor * math.cos(v)) * cx, minor * math.sin(v), (major + minor * math.cos(v)) * cz], np.float32)
        n = np.array([math.cos(v) * cx, math.sin(v), math.cos(v) * cz], np.float32)
        return p, n
    for i in range(nu):
        for j in range(nv):
            (p00, n00), (p10, n10), (p01, n01), (p11, n11) = pt(i, j), pt(i + 1, j), pt(i, j + 1), pt(i + 1, j + 1)
            tris.append(tri36([p00, p10, p11], [n00, n10, n11]))
            tris.append(tri36([p00, p11, p01], [n00, n11, n01]))
    return tris


def dungeon(width=1920, height=1080, mode=MODE_IMAGE, denoise=True, seed=7, cells=13):
    """A *synthetic* dungeon (small parity cases and golden fixtures; the benchmark's C3 is `demo_level` below).

    The reference's demo level (bevy-strolle/assets/demo.zip, 8,393 triangles + 3 emissive tori, 6 point
    lights, sun az 3.0 / alt 0.35, bevy-strolle/examples/demo.rs:150-237) needs the texture atlas (SURVEY
    §8f-3, a "next" row); this generator builds an untextured level of the same scale procedurally: a grid of
    4 m cells with floor/ceiling slabs, random partition walls, pillars and crates (boxes), an open corridor in
    front of the camera, 3 emissive tori, 6 point lights, the same sun, the same camera pose
    (eye (-5.75, 0.5, -16.8) looking down -Z).  Some ceiling slabs are missing so that the sky is visible.
    """
    rng = np.random.RandomState(seed)
    meshes, materials, instances, lights = {}, {}, [], []
    palette = [(0.55, 0.5, 0.45, 1), (0.4, 0.38, 0.36, 1), (0.5, 0.3, 0.2, 1), (0.3, 0.35, 0.4, 1), (0.6, 0.55, 0.4, 1)]
    for i, col in enumerate(palette):
        materials[100 + i] = (material(col, perceptual_roughness=1.0, reflectance=0.0), False)
    materials[150] = (material((0.9, 0.6, 0.3, 1), emissive=(9.0, 6.0, 3.0, 1.0), perceptual_roughness=1.0, reflectance=0.0), False)
    nid = [0]

    def add(tris, mat, xf=IDENTITY_AFFINE):
        h = nid[0]
        nid[0] += 1
        meshes[1000 + h] = np.stack(tris)
        instances.append((5000 + h, 1000 + h, mat, np.asarray(xf, np.float32)))

    S, wall_h = 4.0, 3.0
    eye = np.array([-5.75, 0.5, -16.8])
    half = cells // 2
    # cell (i, j) spans x in [cx(i), cx(i)+S), z in [cz(j), cz(j)+S); the camera sits in the middle of cell (half, half)
    cx = lambda i: eye[0] - S / 2 + (i - half) * S
    cz = lambda j: eye[2] - S / 2 + (j - half) * S
    corridor = {(half, j) for j in range(max(half - 5, 0), half + 1)}
    for i in range(cells):
        for j in range(cells):
            x0, z0 = cx(i), cz(j)
            add(_box((x0, -0.2, z0), (x0 + S, 0.0, z0 + S)), 100 + (i + j) % 2)
            if rng.rand() < 0.85:
                add(_box((x0, wall_h, z0), (x0 + S, wall_h + 0.2, z0 + S)), 101)
            # partition walls on the -z and -x borders, never across the corridor
            if (i, j) not in corridor or (i, j - 1) not in corridor:
                if rng.rand() < 0.4 and not ((i, j) in corridor and (i, j - 1) in corridor):
                    add(_box((x0, 0.0, z0), (x0 + S, wall_h, z0 + 0.3)), 102 + rng.randint(0, 3))
            if (i, j) not in corridor and (i - 1, j) not in corridor and rng.rand() < 0.4:
                add(_box((x0, 0.0, z0), (x0 + 0.3, wall_h, z0 + S)), 102 + rng.randint(0, 3))
            if (i, j) in corridor:
                for side in (-1, 1):   # crates along the corridor sides
                    if rng.rand() < 0.6:
                        px, pz = x0 + S / 2 + side * 1.5, z0 + rng.rand() * (S - 1) + 0.5
                        hgt = 0.3 + rng.rand() * 0.9
                        add(_box((px - 0.25, 0.0, pz - 0.25), (px + 0.25, hgt, pz + 0.25)), 102 + rng.randint(0, 3))
                continue
            for _ in range(rng.randint(0, 4)):
                px, pz = x0 + rng.rand() * (S - 1) + 0.5, z0 + rng.rand() * (S - 1) + 0.5
                hgt = 0.3 + rng.rand() * 1.2
                add(_box((px - 0.25, 0.0, pz - 0.25), (px + 0.25, hgt, pz + 0.25)), 102 + rng.randint(0, 3))
            if rng.rand() < 0.3:
                px, pz = x0 + S / 2, z0 + S / 2
                add(_box((px - 0.2, 0.0, pz - 0.2), (px + 0.2, wall_h, pz + 0.2)), 103)
    lo, hi = cx(0), cx(cells)
    zlo, zhi = cz(0), cz(cells)
    add(_box((lo - 0.3, 0.0, zlo), (lo, wall_h, zhi)), 104); add(_box((hi, 0.0, zlo), (hi + 0.3, wall_h, zhi)), 104)
    add(_box((lo, 0.0, zlo - 0.3), (hi, wall_h, zlo)), 104); add(_box((lo, 0.0, zhi), (hi, wall_h, zhi + 0.3)), 104)
    torus = _torus()
    for k, (dx, dz) in enumerate([(0.0, -6.0), (4.0, -9.0), (-4.0, -12.0)]):
        xf = np.array([0.5, 0, 0, 0, 0.5, 0, 0, 0, 0.5, eye[0] + dx, 1.2, eye[2] + dz], np.float32)
        add(torus, 150, xf)
    inten = 120.0 / (4.0 * math.pi)
    for k, (dx, dz) in enumerate([(0.0, -3.0), (4.5, -7.0), (-4.5, -7.0), (0.0, -13.0), (8.0, -2.0), (-8.0, -2.0)]):
        lights.append((9000 + k, LIGHT_POINT, point_light((eye[0] + dx, 2.4, eye[2] + dz), 0.15, (inten,) * 3, 35.0)))
    cam = dict(mode=mode, denoise=denoise, ref_depth=1, w=width, h=height,
               transform=look_at_transform(tuple(eye), (eye[0], eye[1], eye[2] - 0.2)),
               projection=perspective_infinite_reverse_rh(math.pi / 4.0, width / height, 0.1))
    return dict(name="dungeon_synthetic", meshes=meshes, materials=materials, instances=instances, lights=lights, sun=(3.0, 0.35), camera=cam)


def _bevy_torus(radius=1.0, ring_radius=0.5, segments=32, sides=24):
    """bevy 0.12.1 `shape::Torus::default()` (third-party crate pinned in Cargo.toml:16, not vendored under /root/reference; restated
    from its published mesh generator): (segments+1) x (sides+1) vertices, two triangles (lt, rt, lb), (rt, rb, lb) per face."""
    pos, nor, uvs = [], [], []
    seg_stride, side_stride = np.float32(2.0 * math.pi) / np.float32(segments), np.float32(2.0 * math.pi) / np.float32(sides)
    for seg in range(segments + 1):
        theta = float(seg_stride * np.float32(seg))
        for side in range(sides + 1):
            phi = float(side_stride * np.float32(side))
            p = np.array([math.cos(theta) * (radius + ring_radius * math.cos(phi)), ring_radius * math.sin(phi),
                          math.sin(theta) * (radius + ring_radius * math.cos(phi))], np.float64)
            c = np.array([radius * math.cos(theta), 0.0, radius * math.sin(theta)], np.float64)
            n = (p - c) / np.linalg.norm(p - c)
            pos.append(p.astype(np.float32)); nor.append(n.astype(np.float32)); uvs.append([seg / segments, side / sides])
    tris = []
    row = sides + 1
    for seg in range(segments):
        for side in range(sides):
            lt, rt, lb, rb = side + seg * row, side + 1 + seg * row, side + (seg + 1) * row, side + 1 + (seg + 1) * row
            for a, b, c in ((lt, rt, lb), (rt, rb, lb)):
                tris.append(tri36([pos[a], pos[b], pos[c]], [nor[a], nor[b], nor[c]], [uvs[a], uvs[b], uvs[c]]))
    return tris


def demo_level(width=1920, height=1080, mode=MODE_IMAGE, denoise=True, textures=True):
    """BASELINE config C3: the reference's dungeon demo (bevy-strolle/examples/demo.rs).

    Geometry, materials and textures come from the reference's own asset (assets/demo.zip -> demo/level.glb, extracted
    by tools/make_assets.py into assets/dungeon.npz: 45 meshes, 8,393 triangles, 45 64x64 base-colour textures); the
    rest follows demo.rs: every material re-lit with reflectance 0 / perceptual_roughness 1 (`adjust_materials`,
    demo.rs:246-261 — it walks ALL StandardMaterials, the tori's included), three emissive tori
    (shape::Torus::default(), rotation_z(1.0), scale 0.5, emissive 10 x (0.9, 0.6, 0.3), demo.rs:195-219), six point
    lights of intensity 5000 (x 1/4pi in bevy-strolle/src/stages/extract.rs:285), range 35, radius 0.15 (demo.rs:169-191), the
    flashlight dropped for its zero intensity (extract.rs:306-311), camera eye (-5.75, 0.5, -16.8) -> (-5.75, 0.5, -17.0)
    (demo.rs:150-152), sun azimuth 3.0 (_common.rs:166-173) and strolle::Sun's default altitude 0.35 (strolle/src/sun.rs:7-13).
    `textures=False` is demo.rs's T key (base_color_texture = None on every material)."""
    d = np.load(os.path.join(_ASSETS, "dungeon.npz"))
    meshes, materials, instances, lights, images, material_textures = {}, {}, [], [], {}, {}
    nmesh = len(d["mesh_material"])
    zeros_t = np.zeros((3, 4), np.float32)
    for k in range(nmesh):
        pos, nor, uv = d[f"pos{k}"], d[f"nor{k}"], d[f"uv{k}"]
        tris = np.concatenate([pos.reshape(-1, 9), nor.reshape(-1, 9), uv.reshape(-1, 6), np.tile(zeros_t.reshape(1, 12), (len(pos), 1))], axis=1).astype(np.float32)
        meshes[1000 + k] = tris
        instances.append((5000 + k, 1000 + k, 100 + int(d["mesh_material"][k]), affine_from_colmajor4x4(d["mesh_transform_colmajor"][k])))
    for i, bmr in enumerate(d["material_base_metallic_roughness"]):
        # bevy_gltf StandardMaterial (base colour factor, metallic factor) then demo.rs::adjust_materials: reflectance 0, roughness 1
        materials[100 + i] = (material(tuple(float(v) for v in bmr[:4]), perceptual_roughness=1.0, metallic=float(bmr[4]), reflectance=0.0), False)
        t = int(d["material_texture"][i])
        if textures and t >= 0:
            material_textures[100 + i] = dict(base_color=700 + t)
    if textures:
        for t, img in enumerate(d["images_rgba8"]):
            images[700 + t] = np.ascontiguousarray(img)
    torus = np.stack(_bevy_torus())
    meshes[2000] = torus
    c1, s1 = math.cos(1.0), math.sin(1.0)   # Quat::from_rotation_z(1.0) * scale 0.5
    for k, (tx, ty, tz) in enumerate([(-0.5, 0.33, -5.5), (-11.0, 0.33, 28.0), (-11.5, 0.33, 13.5)]):
        materials[160 + k] = (material((0.9, 0.6, 0.3, 1.0), emissive=(9.0, 6.0, 3.0, 1.0), perceptual_roughness=1.0, reflectance=0.0), False)
        xf = np.array([0.5 * c1, 0.5 * s1, 0.0, -0.5 * s1, 0.5 * c1, 0.0, 0.0, 0.0, 0.5, tx, ty, tz], np.float32)
        instances.append((6000 + k, 2000, 160 + k, xf))
    inten = 5000.0 / (4.0 * math.pi)
    for k, p in enumerate([(-3.0, 0.75, -23.0), (-23.5, 0.75, -31.0), (1.25, 0.75, -10.5), (-3.15, 0.75, 1.25), (-3.25, 0.75, 20.25), (13.25, 0.75, -28.25)]):
        lights.append((9000 + k, LIGHT_POINT, point_light(p, 0.15, (inten,) * 3, 35.0)))
    cam = dict(mode=mode, denoise=denoise, ref_depth=1, w=width, h=height,
               transform=look_at_transform((-5.75, 0.5, -16.8), (-5.75, 0.5, -17.0)),
               projection=perspective_infinite_reverse_rh(math.pi / 4.0, width / height, 0.1))
    return dict(name="dungeon_demo_level", meshes=meshes, materials=materials, instances=instances, lights=lights, sun=(3.0, 0.35), camera=cam,
                images=images, material_textures=material_textures)


DEMO_TORI = (6000, 6001, 6002)   # demo_level's torus instances
_DEMO_TORUS_AT = [(-0.5, 0.33, -5.5), (-11.0, 0.33, 28.0), (-11.5, 0.33, 13.5)]


def _quat_mul(a, b):
    (aw, ax, ay, az), (bw, bx, by, bz) = a, b
    return (aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
            aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw)


def _affine_trs(q, scale, t):
    """Transform::from_translation(t).with_rotation(q).with_scale(scale) as 12 floats (matrix columns x, y, z, translation)."""
    w, x, y, z = q
    cols = [(1 - 2 * (y * y + z * z), 2 * (x * y + w * z), 2 * (x * z - w * y)),
            (2 * (x * y - w * z), 1 - 2 * (x * x + z * z), 2 * (y * z + w * x)),
            (2 * (x * z + w * y), 2 * (y * z - w * x), 1 - 2 * (x * x + y * y))]
    return np.array([c * s for col, s in zip(cols, scale) for c in col] + list(t), np.float32)


def demo_level_animated(t):
    """The tori of demo_level at time `t` (seconds) as bevy-strolle/examples/demo.rs `animate_toruses` turns them:
    rotation = Quat::from_rotation_z(t) * Quat::from_rotation_x(t + 1), scale 0.5, translation unchanged.  Returns
    (instance, mesh, material, affine12) tuples to re-insert; every other instance of demo_level stays where it is."""
    rz = (math.cos(0.5 * t), 0.0, 0.0, math.sin(0.5 * t))
    rx = (math.cos(0.5 * (t + 1.0)), math.sin(0.5 * (t + 1.0)), 0.0, 0.0)
    q = _quat_mul(rz, rx)
    return [(h, 2000, 160 + k, _affine_trs(q, (0.5, 0.5, 0.5), at)) for k, (h, at) in enumerate(zip(DEMO_TORI, _DEMO_TORUS_AT))]


def _icosphere(subdivisions=1):
    """A unit icosphere (20 * 4^subdivisions triangles, flat-free vertex normals = positions)."""
    p = (1 + 5 ** 0.5) / 2
    v = [np.array(a, np.float64) for a in ((-1, p, 0), (1, p, 0), (-1, -p, 0), (1, -p, 0), (0, -1, p), (0, 1, p), (0, -1, -p), (0, 1, -p),
                                            (p, 0, -1), (p, 0, 1), (-p, 0, -1), (-p, 0, 1))]
    v = [a / np.linalg.norm(a) for a in v]
    faces = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2), (10, 7, 6), (7, 1, 8),
             (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11), (6, 2, 10), (8, 6, 7), (9, 8, 1)]
    tris = [tuple(v[i] for i in f) for f in faces]
    for _ in range(subdivisions):
        nxt = []
        for a, b, c in tris:
            ab, bc, ca = [m / np.linalg.norm(m) for m in ((a + b) / 2, (b + c) / 2, (c + a) / 2)]
            nxt += [(a, ab, ca), (b, bc, ab), (c, ca, bc), (ab, bc, ca)]
        tris = nxt
    return [tri36([a, b, c], [a, b, c]) for a, b, c in tris]


STRESS_FLOOR = 7000   # stress_bvh's floor instance; its objects are 7001 .. 7000 + n


def stress_bvh_instances(n, t):
    """The `n` objects of stress_bvh at time `t`: object k (a unit box for even k, an icosphere of radius 0.5 for odd k) circles
    its own spot on the floor, bounces and tumbles on a scripted path (no physics, fully deterministic)."""
    out = []
    for k in range(n):
        r = 3.0 + 40.0 * ((k * 0.6180339887) % 1.0)
        a0 = 2.0 * math.pi * ((k * 0.7548776662) % 1.0)
        a = a0 + 0.3 * t / (1.0 + 0.05 * r)
        y = 1.0 + 0.5 * (k % 7) + 2.0 * abs(math.sin(1.3 * t + k))
        spin = 0.9 * t + k
        q = _quat_mul((math.cos(0.5 * spin), 0.0, math.sin(0.5 * spin), 0.0), (math.cos(0.25 * spin), math.sin(0.25 * spin), 0.0, 0.0))
        s = 1.0 if k % 2 == 0 else 0.5
        out.append((STRESS_FLOOR + 1 + k, 201 if k % 2 == 0 else 202, 101 + k % 3, _affine_trs(q, (s, s, s), (r * math.cos(a), y, r * math.sin(a)))))
    return out


def stress_bvh(n=2000, width=1920, height=1080, mode=MODE_IMAGE, denoise=True, t=0.0):
    """A scene shaped like bevy-strolle/examples/stress-bvh.rs: a 100 x 1 x 100 floor box and `n` unit boxes and icospheres
    (20 triangles, where the example's shape::Icosphere::default() has 20480) that move every tick along the
    scripted paths of stress_bvh_instances instead of the example's physics."""
    meshes = {200: np.stack(_box((-50.0, -1.0, -50.0), (50.0, 0.0, 50.0))), 201: np.stack(_box((-0.5, -0.5, -0.5), (0.5, 0.5, 0.5))),
              202: np.stack(_icosphere(0))}
    materials = {100: (material((0.6, 0.6, 0.6, 1.0)), False), 101: (material((0.8, 0.3, 0.2, 1.0)), False),
                 102: (material((0.2, 0.5, 0.8, 1.0)), False), 103: (material((0.3, 0.7, 0.3, 1.0), perceptual_roughness=0.5), False)}
    instances = [(STRESS_FLOOR, 200, 100, IDENTITY_AFFINE)] + stress_bvh_instances(n, t)
    lights = [(400, LIGHT_POINT, point_light((0.0, 12.0, 0.0), 0.3, (400.0, 400.0, 400.0), 60.0))]
    cam = dict(mode=mode, denoise=denoise, ref_depth=1, w=width, h=height, transform=look_at_transform((0.0, 22.0, 48.0), (0.0, 0.0, 0.0)),
               projection=perspective_infinite_reverse_rh(math.pi / 4.0, width / height, 0.1))
    return dict(name="stress_bvh", meshes=meshes, materials=materials, instances=instances, lights=lights, sun=(1.0, 0.6), camera=cam)


def _hsl_linear(h, s, l):
    """Bevy's Color::hsl(h, s, l).as_linear_rgba_f32() for the rgb part: HSL -> sRGB, then the sRGB transfer curve."""
    c = (1.0 - abs(2.0 * l - 1.0)) * s
    hp = (h % 360.0) / 60.0
    x = c * (1.0 - abs(hp % 2.0 - 1.0))
    r, g, b = [(c, x, 0), (x, c, 0), (0, c, x), (0, x, c), (x, 0, c), (c, 0, x)][min(int(hp), 5)]
    m = l - c / 2.0
    lin = lambda v: v / 12.92 if v <= 0.04045 else ((v + 0.055) / 1.055) ** 2.4
    return tuple(lin(v + m) for v in (r, g, b))


STRESS_LIGHTS_FIRST = 400   # stress_lights' light handles: 400 .. 499


def stress_lights_lights(t):
    """The 100 point lights of stress_lights at time `t` (stress-lights.rs update_lights): light k, with phase k * 123.456, circles its
    room's anchor at radius 4 with the angle u = phase * 2 pi + t and takes the hue (u * 90) mod 360; range 20, radius 0.25,
    intensity 3000 (x 1/4pi, as the reference's extract does)."""
    out, phase, inten = [], 0.0, 3000.0 / (4.0 * math.pi)
    k = 0
    for x in range(-5, 5):
        for y in range(10):
            ax, ay = x * 15.0, y * 15.0
            u = phase * 2.0 * math.pi + t
            pos = (ax + 4.0 * math.sin(u), 5.0 + ay + 4.0 * math.cos(u), 0.0)
            col = tuple(v * inten for v in _hsl_linear((u * 90.0) % 360.0, 1.0, 0.5))
            out.append((STRESS_LIGHTS_FIRST + k, LIGHT_POINT, point_light(pos, 0.25, col, 20.0)))
            phase += 123.456
            k += 1
    return out


def stress_lights(width=512, height=512, mode=MODE_IMAGE, denoise=True, ref_depth=1, t=0.0):
    """bevy-strolle/examples/stress-lights.rs: a 1000 x 1 x 1000 floor box at y = -2 and a 10 x 10 grid of rooms 15 apart (five
    scaled unit boxes each: two side walls, a back wall, a ceiling and a floor), each with a moving, recolouring point light of
    range 20 (stress_lights_lights); sun altitude -1, camera (0, 50, 80) -> (0, 50, 0).  `t` is the example's elapsed time."""
    walls = [((1.0, 10.0, 10.0), (-5.0, 5.0, 0.0)), ((1.0, 10.0, 10.0), (5.0, 5.0, 0.0)), ((10.0, 10.0, 1.0), (0.0, 5.0, -5.0)),
             ((10.0, 1.0, 10.0), (0.0, 10.0, 0.0)), ((10.0, 1.0, 10.0), (0.0, 0.0, 0.0))]
    scaled = lambda sc, tr: np.array([sc[0], 0, 0, 0, sc[1], 0, 0, 0, sc[2], tr[0], tr[1], tr[2]], np.float32)
    instances = [(300, 200, 100, scaled((1000.0, 1.0, 1000.0), (0.0, -2.0, 0.0)))]
    h = 301
    for x in range(-5, 5):
        for y in range(10):
            for sc, tr in walls:
                instances.append((h, 200, 100, scaled(sc, (tr[0] + x * 15.0, tr[1] + y * 15.0, tr[2]))))
                h += 1
    cam = dict(mode=mode, denoise=denoise, ref_depth=ref_depth, w=width, h=height,
               transform=look_at_transform((0.0, 50.0, 80.0), (0.0, 50.0, 0.0)),
               projection=perspective_infinite_reverse_rh(math.pi / 4.0, width / height, 0.1))
    return dict(name="stress_lights", meshes={200: np.stack(_box((-0.5, -0.5, -0.5), (0.5, 0.5, 0.5)))},
                materials={100: (material((1.0, 1.0, 1.0, 1.0), perceptual_roughness=0.5), False)}, instances=instances, lights=stress_lights_lights(t),
                sun=(0.0, -1.0), camera=cam)


def _quad(p0, p1, p2, p3, normal, uv_lo=(0.0, 0.0), uv_hi=(1.0, 1.0), tangents=None):
    """Two triangles wound so that the geometric normal agrees with `normal` (Triangle::hit flips the shading normal by
    the sign of the determinant, strolle-gpu/src/triangle.rs:95-101, i.e. it trusts the winding).  `tangents`: one
    (x, y, z, handedness) for all four corners; None = zero tangents (a mesh without ATTRIBUTE_TANGENT)."""
    (u0, v0), (u1, v1) = uv_lo, uv_hi
    c = [np.asarray(p, np.float64) for p in (p0, p1, p2, p3)]
    uv = [[u0, v0], [u1, v0], [u1, v1], [u0, v1]]
    if np.dot(np.cross(c[1] - c[0], c[2] - c[0]), np.asarray(normal, np.float64)) < 0:
        c = [c[0], c[3], c[2], c[1]]
        uv = [uv[0], uv[3], uv[2], uv[1]]
    t = None if tangents is None else [tangents] * 3
    return [tri36([c[0], c[1], c[2]], [normal] * 3, [uv[0], uv[1], uv[2]], t), tri36([c[0], c[2], c[3]], [normal] * 3, [uv[0], uv[2], uv[3]], t)]


def textured_room(width=320, height=180, mode=MODE_IMAGE, denoise=True):
    """Exercises the texture atlas (SURVEY §8f-3): sRGB base-colour textures with repeat-wrapped (also negative) uvs,
    an emissive texture, a metallic-roughness texture, and an alpha-cutout AlphaMode::Blend fence whose holes must let
    primary, shadow and bounce rays through (strolle-gpu/src/ray.rs:212-229, material.rs:76-104)."""
    rng = np.random.RandomState(3)
    def checker(n, cell, a, b):
        img = np.zeros((n, n, 4), np.uint8)
        yy, xx = np.mgrid[0:n, 0:n]
        m = ((xx // cell) + (yy // cell)) % 2 == 0
        img[m] = a; img[~m] = b
        return img
    images = {
        700: checker(64, 8, (200, 180, 150, 255), (90, 60, 40, 255)),                      # floor base colour
        701: checker(32, 4, (255, 255, 255, 255), (0, 0, 0, 0)),                             # fence: alpha cutout
        702: (rng.randint(0, 256, size=(16, 48, 4))).astype(np.uint8),                       # emissive noise (non-square)
        703: checker(16, 2, (255, 64, 255, 255), (255, 255, 32, 255)),                       # metallic-roughness (g = roughness, b = metallic)
    }
    images[702][..., 3] = 255
    materials = {
        100: (material((1.0, 1.0, 1.0, 1.0)), False), 101: (material((0.7, 0.7, 0.75, 1.0)), False),
        102: (material((1.0, 1.0, 1.0, 1.0)), True),                                           # fence, AlphaMode::Blend
        103: (material((0.2, 0.2, 0.2, 1.0), emissive=(3.0, 2.0, 1.0, 1.0)), False),
        104: (material((0.9, 0.8, 0.6, 1.0), perceptual_roughness=0.8, metallic=1.0), False),
    }
    material_textures = {100: dict(base_color=700), 102: dict(base_color=701), 103: dict(emissive=702), 104: dict(metallic_roughness=703, base_color=700)}
    meshes = {
        200: np.stack(_quad((-3, 0, -3), (3, 0, -3), (3, 0, 3), (-3, 0, 3), (0, 1, 0), (-1.5, -1.5), (2.5, 2.5))),     # floor, uvs span [-1.5, 2.5]
        201: np.stack(_quad((-3, 0, -3), (-3, 3, -3), (3, 3, -3), (3, 0, -3), (0, 0, 1))),                              # back wall
        202: np.stack(_quad((-1.5, 0, 0.5), (1.5, 0, 0.5), (1.5, 2.0, 0.5), (-1.5, 2.0, 0.5), (0, 0, 1), (0, 0), (3, 2))),  # fence
        203: np.stack(_quad((-3, 0.5, -2.9), (-3, 2.5, -2.9), (-1, 2.5, -2.9), (-1, 0.5, -2.9), (0, 0, 1))),            # emissive panel
        204: np.stack(_box((0.8, 0.0, -1.6), (1.8, 1.0, -0.6))),                                                         # metal box
    }
    instances = [(300, 200, 100, IDENTITY_AFFINE), (301, 201, 101, IDENTITY_AFFINE), (302, 202, 102, IDENTITY_AFFINE),
                 (303, 203, 103, IDENTITY_AFFINE), (304, 204, 104, IDENTITY_AFFINE)]
    lights = [(400, LIGHT_POINT, point_light((0.0, 2.5, 2.0), 0.1, (6.0, 6.0, 6.0), 20.0)), (401, LIGHT_POINT, point_light((-1.0, 1.5, -1.5), 0.1, (2.0, 2.0, 3.0), 20.0))]
    cam = dict(mode=mode, denoise=denoise, ref_depth=1, w=width, h=height, transform=look_at_transform((0.3, 1.2, 4.0), (0.0, 0.9, 0.0)),
               projection=perspective_infinite_reverse_rh(math.pi / 4.0, width / height, 0.1))
    return dict(name="textured_room", meshes=meshes, materials=materials, instances=instances, lights=lights, sun=(1.0, 0.6), camera=cam,
                images=images, material_textures=material_textures)


def tiled_ground(width=320, height=180, mode=MODE_IMAGE, denoise=True, ref_depth=1):
    """Exercises texture filtering (ST_OPT_TEXTURE_FILTER): a large ground plane carrying a 256x256 texture tiled 60 times each way,
    seen at grazing angles (minification up to the last mip levels); a 45x27 (non-power-of-two) textured wall close to the camera
    (magnification); an emissive-textured panel; a metallic-roughness-textured box; and an alpha-cut-out fence."""
    rng = np.random.RandomState(5)
    yy, xx = np.mgrid[0:256, 0:256]
    ground = np.zeros((256, 256, 4), np.uint8)
    m = ((xx // 16) + (yy // 16)) % 2 == 0
    ground[m] = (230, 220, 200, 255); ground[~m] = (40, 60, 90, 255)
    ground[(xx % 64) < 2] = (200, 30, 30, 255)                                       # thin lines: the aliasing a minified fetch shows
    wall = rng.randint(0, 256, size=(27, 45, 4)).astype(np.uint8); wall[..., 3] = 255
    panel = np.zeros((32, 32, 4), np.uint8); panel[..., 3] = 255
    panel[..., 0] = (np.mgrid[0:32, 0:32][1] * 8).astype(np.uint8); panel[..., 1] = 120; panel[..., 2] = (255 - np.mgrid[0:32, 0:32][0] * 8).astype(np.uint8)
    mr = rng.randint(0, 256, size=(8, 8, 4)).astype(np.uint8); mr[..., 3] = 255
    fence = np.zeros((32, 32, 4), np.uint8); fence[...] = (255, 255, 255, 255)
    fence[(np.mgrid[0:32, 0:32][1] % 8) >= 4] = (0, 0, 0, 0)
    images = {720: ground, 721: wall, 722: panel, 723: mr, 724: fence}
    materials = {
        110: (material((1.0, 1.0, 1.0, 1.0)), False), 111: (material((0.9, 0.9, 0.9, 1.0)), False),
        112: (material((0.2, 0.2, 0.2, 1.0), emissive=(2.0, 2.0, 2.0, 1.0)), False),
        113: (material((0.9, 0.8, 0.6, 1.0), perceptual_roughness=0.8, metallic=1.0), False),
        114: (material((0.8, 0.8, 0.8, 1.0)), True),
    }
    material_textures = {110: dict(base_color=720), 111: dict(base_color=721), 112: dict(emissive=722), 113: dict(metallic_roughness=723),
                         114: dict(base_color=724)}
    meshes = {
        210: np.stack(_quad((-60, 0, -60), (60, 0, -60), (60, 0, 60), (-60, 0, 60), (0, 1, 0), (0.0, 0.0), (60.0, 60.0))),   # ground
        211: np.stack(_quad((0.6, 0.2, 2.2), (0.6, 1.4, 2.2), (1.4, 1.4, 3.0), (1.4, 0.2, 3.0), (-1, 0, 1))),                   # wall near the camera
        212: np.stack(_quad((-3, 0.5, -4), (-3, 2.5, -4), (-1, 2.5, -4), (-1, 0.5, -4), (0, 0, 1), (0, 0), (2, 2))),             # emissive panel
        213: np.stack(_box((0.8, 0.0, -1.6), (1.8, 1.0, -0.6))),                                                                 # metal box
        214: np.stack(_quad((-2.5, 0, -1), (-0.5, 0, -1), (-0.5, 1.2, -1), (-2.5, 1.2, -1), (0, 0, 1), (0, 0), (4, 2))),         # fence
    }
    instances = [(310, 210, 110, IDENTITY_AFFINE), (311, 211, 111, IDENTITY_AFFINE), (312, 212, 112, IDENTITY_AFFINE),
                 (313, 213, 113, IDENTITY_AFFINE), (314, 214, 114, IDENTITY_AFFINE)]
    lights = [(410, LIGHT_POINT, point_light((0.0, 3.0, 1.0), 0.1, (8.0, 8.0, 8.0), 30.0))]
    cam = dict(mode=mode, denoise=denoise, ref_depth=ref_depth, w=width, h=height, transform=look_at_transform((0.0, 0.9, 4.0), (0.0, 0.6, -10.0)),
               projection=perspective_infinite_reverse_rh(math.pi / 4.0, width / height, 0.1))
    return dict(name="tiled_ground", meshes=meshes, materials=materials, instances=instances, lights=lights, sun=(1.0, 0.35), camera=cam,
                images=images, material_textures=material_textures)


def brick_normal_map(n=64, rows=4, cols=2, mortar=0.06, bevel=0.05, seed=11):
    """A brick-wall tangent-space normal map (RGBA8, n x n, linear bytes 255 (t + 1) / 2): bevelled bricks in running bond,
    flat mortar joints, a little per-brick tilt and grain, and one 6 x 6 patch whose texels point below the surface
    (t.z < 0), which the shading rule falls back from."""
    rng = np.random.RandomState(seed)
    yy, xx = (np.mgrid[0:n, 0:n] + 0.5) / n
    row = np.floor(yy * rows)
    xs = xx * cols + 0.5 * (row % 2)
    fx, fy = xs - np.floor(xs), yy * rows - row
    brick = (row * 2 * cols + np.floor(xs)).astype(np.int64) % (2 * cols * rows)
    tilt = rng.uniform(-0.15, 0.15, size=(2 * cols * rows, 2))
    t = np.zeros((n, n, 3))
    t[..., 0], t[..., 1] = tilt[brick, 0], tilt[brick, 1]
    # bevels: the normal leans outwards over the last `bevel` of each brick edge
    for f, k, s in ((fx, 0, 1.0), (fy, 1, 1.0)):
        t[..., k] += np.where(f < mortar + bevel, -0.6 * s, 0.0) + np.where(f > 1.0 - bevel, 0.6 * s, 0.0)
    joint = (fx < mortar) | (fy < mortar)
    t[..., 0] = np.where(joint, 0.0, t[..., 0]); t[..., 1] = np.where(joint, 0.0, t[..., 1])
    t[..., :2] += rng.normal(scale=0.04, size=(n, n, 2))
    t[..., 2] = 1.0
    t /= np.linalg.norm(t, axis=-1, keepdims=True)
    t[n // 2:n // 2 + 6, n // 2:n // 2 + 6] = (0.1, -0.2, -0.97)
    img = np.full((n, n, 4), 255, np.uint8)
    img[..., :3] = np.clip(np.round((t + 1.0) * 127.5), 0, 255).astype(np.uint8)
    return img


def ripple_normal_map(n=32, waves=3):
    """Sinusoidal ridges along u (RGBA8 tangent-space normal map)."""
    u = (np.arange(n) + 0.5) / n
    sx = 0.5 * np.sin(2 * np.pi * waves * u)
    t = np.stack(np.broadcast_arrays(sx[None, :], np.zeros((n, 1)), np.ones((n, n))), axis=-1)
    t /= np.linalg.norm(t, axis=-1, keepdims=True)
    img = np.full((n, n, 4), 255, np.uint8)
    img[..., :3] = np.clip(np.round((t + 1.0) * 127.5), 0, 255).astype(np.uint8)
    return img


def _tangent_torus(major=0.5, minor=0.2, nu=32, nv=16, tile=(4.0, 2.0)):
    """A torus with per-vertex uvs and analytic tangents (dP/du, handedness from dP/dv): the tangent turns along the
    surface, so the interpolated, not renormalised, tangent of a triangle is shorter than 1."""
    tris = []
    def vert(i, j):
        a, b = 2 * math.pi * i / nu, 2 * math.pi * j / nv
        ca, sa, cb, sb = math.cos(a), math.sin(a), math.cos(b), math.sin(b)
        p = np.array([(major + minor * cb) * ca, minor * sb, (major + minor * cb) * sa])
        n = np.array([cb * ca, sb, cb * sa])
        t = np.array([-sa, 0.0, ca])
        dv = np.array([-sb * ca, cb, -sb * sa])
        w = 1.0 if np.dot(np.cross(n, t), dv) >= 0 else -1.0
        return p, n, [tile[0] * i / nu, tile[1] * j / nv], list(t) + [w]
    for i in range(nu):
        for j in range(nv):
            v00, v10, v01, v11 = vert(i, j), vert(i + 1, j), vert(i, j + 1), vert(i + 1, j + 1)
            for a, b, c in ((v00, v01, v11), (v00, v11, v10)):
                tris.append(tri36([a[0], b[0], c[0]], [a[1], b[1], c[1]], [a[2], b[2], c[2]], [a[3], b[3], c[3]]))
    return tris


def normal_mapped_room(width=224, height=126, mode=MODE_IMAGE, denoise=True, ref_depth=1):
    """Normal maps (ST_OPT_NORMAL_MAPS): a brick-mapped floor and back wall, a ripple-mapped torus with analytic tangents and
    a mirrored copy of it (negative determinant: the baked handedness flips), a brick-mapped two-sided panel seen from
    behind, a brick-mapped box without tangents (NaN tangents: the interpolated normal stays) and an unmapped box.  All
    dielectric with perceptual roughness >= 0.5, and the sun below the horizon: the fast-shading tier's drift from the strict tier on
    sunlit direct light (2.7e-3 relative L2 on the textured room's first frame on an H100, maps or not) would blur the 1e-3
    product-tier check.  Instance 304 (the torus) is the one the tests move."""
    images = {710: brick_normal_map(), 711: ripple_normal_map()}
    materials = {
        100: (material((0.8, 0.7, 0.6, 1.0), perceptual_roughness=0.6), False),      # floor, brick map
        101: (material((0.7, 0.45, 0.35, 1.0), perceptual_roughness=0.8), False),    # back wall / panel / box without tangents, brick map
        102: (material((0.5, 0.6, 0.8, 1.0), perceptual_roughness=0.5), False),      # tori, ripple map
        103: (material((0.6, 0.65, 0.6, 1.0), perceptual_roughness=0.9), False),     # no normal map
    }
    material_textures = {100: dict(normal_map=710), 101: dict(normal_map=710), 102: dict(normal_map=711)}
    meshes = {
        200: np.stack(_quad((-3, 0, -3), (3, 0, -3), (3, 0, 3), (-3, 0, 3), (0, 1, 0), (0, 0), (3, 3), tangents=(1, 0, 0, -1))),
        201: np.stack(_quad((-3, 0, -3), (-3, 3, -3), (3, 3, -3), (3, 0, -3), (0, 0, 1), (0, 0), (3, 1.5), tangents=(1, 0, 0, 1))),
        202: np.stack(_quad((-2.4, 0.2, 0.6), (-1.4, 0.2, 0.6), (-1.4, 1.4, 0.6), (-2.4, 1.4, 0.6), (0, 0, -1), (0, 0), (1, 1), tangents=(-1, 0, 0, 1))),
        203: np.stack(_box((0.9, 0.0, -1.9), (1.7, 0.8, -1.1))),
        204: np.stack(_tangent_torus()),
        205: np.stack(_box((-1.8, 0.0, -2.2), (-1.1, 0.6, -1.5))),
    }
    instances = [(300, 200, 100, IDENTITY_AFFINE), (301, 201, 101, IDENTITY_AFFINE), (302, 202, 101, IDENTITY_AFFINE),
                 (303, 203, 101, IDENTITY_AFFINE),
                 (304, 204, 102, np.array([1, 0, 0, 0, 0, 1, 0, -1, 0, -0.3, 0.7, -0.6], np.float32)),     # stood up, facing the camera
                 (305, 204, 102, np.array([-1, 0, 0, 0, 1, 0, 0, 0, 1, 1.6, 0.25, 0.2], np.float32)),     # mirrored in x, lying down
                 (306, 205, 103, IDENTITY_AFFINE)]
    lights = [(400, LIGHT_POINT, point_light((0.5, 2.4, 1.5), 0.1, (6.0, 6.0, 6.0), 20.0)),
              (401, LIGHT_POINT, point_light((-1.5, 1.2, -0.5), 0.1, (2.0, 2.0, 3.0), 20.0))]
    cam = dict(mode=mode, denoise=denoise, ref_depth=ref_depth, w=width, h=height, transform=look_at_transform((0.4, 1.5, 3.8), (0.0, 0.6, -0.5)),
               projection=perspective_infinite_reverse_rh(math.pi / 4.0, width / height, 0.1))
    return dict(name="normal_mapped_room", meshes=meshes, materials=materials, instances=instances, lights=lights, sun=(1.0, -1.0), camera=cam,
                images=images, material_textures=material_textures)


def apply(engine, scene):
    """Feed a scene through the Engine API in a fixed order; returns the camera handle."""
    for h, rgba in scene.get("images", {}).items():
        engine.insert_image(h, rgba)
    for h, tris in scene["meshes"].items():
        engine.insert_mesh(h, tris)
    for h, (params, alpha) in scene["materials"].items():
        engine.insert_material(h, params, alpha)
    for h, tex in scene.get("material_textures", {}).items():
        engine.set_material_textures(h, **tex)
    for h, mesh, mat, xf in scene["instances"]:
        engine.insert_instance(h, mesh, mat, xf)
    for h, kind, params in scene["lights"]:
        engine.insert_light(h, kind, params)
    engine.update_sun(*scene["sun"])
    if "environment_map" in scene:
        engine.set_environment_map(**scene["environment_map"])
    c = scene["camera"]
    return engine.create_camera(c["mode"], c["denoise"], c["ref_depth"], c["w"], c["h"], c["transform"], c["projection"])


def aa_edges(width=96, height=64, mode=MODE_IMAGE, denoise=True, ref_depth=1):
    """Measures anti-aliasing (ST_OPT_TEMPORAL_AA): a black (albedo 0, metallic 0, reflectance 0) backdrop filling the view, and in front
    of it, 0.1 units off the backdrop, an emissive quad rotated by 0.3 rad about the view axis and an emissive bar 0.3 pixels wide and
    tilted by 0.05 rad.  No lights, the sun below the horizon: every composed pixel is exactly an emissive colour or 0, so the frame is
    free of noise and its edges are the only signal.  The camera at the origin looks down -z; the backdrop is at z = -5."""
    black = material((0.0, 0.0, 0.0, 1.0), reflectance=0.0)
    materials = {120: (black, False),
                 121: (material((0.0, 0.0, 0.0, 1.0), emissive=(1.0, 0.6, 0.3, 1.0), reflectance=0.0), False),
                 122: (material((0.0, 0.0, 0.0, 1.0), emissive=(0.4, 0.8, 1.0, 1.0), reflectance=0.0), False)}
    z, zf = -5.0, -4.9
    px = 2.0 * -zf * math.tan(math.pi / 8.0) / height   # one pixel at the depth of the emissive shapes

    def rotated(cx, cy, hw, hh, a, zz):
        c, s = math.cos(a), math.sin(a)
        pts = [(cx + c * x - s * y, cy + s * x + c * y, zz) for x, y in ((-hw, -hh), (hw, -hh), (hw, hh), (-hw, hh))]
        return np.stack(_quad(*pts, (0, 0, 1)))
    meshes = {220: np.stack(_quad((-20, -20, z), (20, -20, z), (20, 20, z), (-20, 20, z), (0, 0, 1))),
              221: rotated(-0.35 * px * width, 0.0, 0.25 * px * width, 0.3 * px * height, 0.3, zf),
              222: rotated(0.3 * px * width, 0.0, 0.15 * px, 0.4 * px * height, 0.05, zf)}
    instances = [(320, 220, 120, IDENTITY_AFFINE), (321, 221, 121, IDENTITY_AFFINE), (322, 222, 122, IDENTITY_AFFINE)]
    cam = dict(mode=mode, denoise=denoise, ref_depth=ref_depth, w=width, h=height, transform=look_at_transform((0.0, 0.0, 0.0), (0.0, 0.0, -1.0)),
               projection=perspective_infinite_reverse_rh(math.pi / 4.0, width / height, 0.1))
    return dict(name="aa_edges", meshes=meshes, materials=materials, instances=instances, lights=[], sun=(0.0, -1.0), camera=cam)


def courtyard_sky(width=256, height=128, sun_disc=True):
    """An equirectangular test sky (height x width x 4 linear RGB, row 0 the zenith), generated rather than loaded: a horizon gradient
    (bright near the horizon, deep blue at the zenith, dark brown below), tinted by one colour per azimuth quadrant, and a small disc
    of radiance ~50 (a firefly source, placed so that it straddles the u = 0 / 1 seam)."""
    v = (np.arange(height, dtype=np.float64) + 0.5) / height
    u = (np.arange(width, dtype=np.float64) + 0.5) / width
    uu, vv = np.meshgrid(u, v)
    alt = 0.5 - vv   # +0.5 at the zenith, -0.5 at the nadir (in units of pi)
    sky = np.where(alt[..., None] >= 0, (1.0 - 2.0 * alt[..., None]) * np.array([1.1, 1.0, 0.9]) + 2.0 * alt[..., None] * np.array([0.15, 0.3, 0.9]),
                   np.array([0.25, 0.18, 0.12]) * (1.0 + 2.0 * alt[..., None]))
    quadrant = np.floor(uu * 4.0).astype(int) % 4
    tint = np.array([[1.0, 0.85, 0.85], [0.85, 1.0, 0.85], [0.85, 0.85, 1.0], [1.0, 1.0, 0.8]])[quadrant]
    rgb = sky * tint
    if sun_disc:
        # the disc: centred on the seam (u = 0), 20 degrees above the horizon, 4 degrees across
        du = np.minimum(uu, 1.0 - uu) * 2.0 * math.pi
        dv = (vv - (0.5 - 20.0 / 180.0)) * math.pi
        rgb[(du * du + dv * dv) < math.radians(2.0) ** 2] = (50.0, 47.0, 42.0)
    out = np.ones((height, width, 4), np.float32)
    out[..., :3] = rgb
    return out


def env_courtyard_motion(t):
    """Frame t's camera transform and moving-crate affine for env_courtyard: the camera orbits slowly, the crate slides."""
    a = 0.05 * t
    eye = (3.5 * math.sin(a), 1.4, 3.5 * math.cos(a))
    crate = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, -0.8 + 0.07 * t, 0.0, 0.6], np.float32)
    return look_at_transform(eye, (0.0, 0.8, 0.0)), crate


def env_courtyard(width=320, height=180, mode=MODE_IMAGE, denoise=True, ref_depth=1):
    """Exercises the environment map (st_set_environment_map): a ground plane and a few occluders (two walls, a pillar, a crate that
    moves), open to the sky, lit by one dim point light and the map (`environment_map`: courtyard_sky at intensity 1.5).  The sun is
    below the horizon (altitude -1.2): the map is the only sky light, and K13's sky-draw probability would be 0 without a map."""
    materials = {130: (material((0.55, 0.5, 0.45, 1.0)), False), 131: (material((0.8, 0.75, 0.7, 1.0), perceptual_roughness=0.6), False),
                 132: (material((0.3, 0.35, 0.5, 1.0), perceptual_roughness=0.3, metallic=0.8), False),
                 133: (material((0.7, 0.4, 0.2, 1.0)), False)}
    meshes = {230: np.stack(_quad((-20, 0, -20), (20, 0, -20), (20, 0, 20), (-20, 0, 20), (0, 1, 0))),
              231: np.stack(_box((-2.5, 0.0, -2.2), (1.5, 1.8, -1.9))),
              232: np.stack(_box((1.9, 0.0, -2.0), (2.2, 1.2, 1.0))),
              233: np.stack(_box((-0.2, 0.0, -0.9), (0.2, 2.4, -0.5))),
              234: np.stack(_box((-0.35, 0.0, -0.35), (0.35, 0.7, 0.35)))}
    cam_xf, crate = env_courtyard_motion(0)
    instances = [(330, 230, 130, IDENTITY_AFFINE), (331, 231, 131, IDENTITY_AFFINE), (332, 232, 131, IDENTITY_AFFINE),
                 (333, 233, 132, IDENTITY_AFFINE), (334, 234, 133, crate)]
    lights = [(430, LIGHT_POINT, point_light((-1.0, 2.0, 1.0), 0.1, (1.5, 1.4, 1.2), 15.0))]
    cam = dict(mode=mode, denoise=denoise, ref_depth=ref_depth, w=width, h=height, transform=cam_xf,
               projection=perspective_infinite_reverse_rh(math.pi / 3.0, width / height, 0.1))
    return dict(name="env_courtyard", meshes=meshes, materials=materials, instances=instances, lights=lights, sun=(0.0, -1.2), camera=cam,
                environment_map=dict(rgba=courtyard_sky(), intensity=1.5, rotation=0.0))


def sunlit_sky(width=2048, height=1024, sun_radiance=2.0e5, sun_altitude_deg=40.0, sun_u=0.3):
    """An equirectangular test sky (height x width x 4 linear RGB, row 0 the zenith) for environment-map sampling: a dim gradient
    (about 0.2 to 0.5 above the horizon, a dark ground below) and a sun disc 0.5 degrees across of radiance `sun_radiance` at
    `sun_altitude_deg` and column `sun_u`.  At the defaults the disc carries about 90% of the irradiance of an open horizontal
    surface."""
    v = (np.arange(height, dtype=np.float64) + 0.5) / height
    u = (np.arange(width, dtype=np.float64) + 0.5) / width
    uu, vv = np.meshgrid(u, v)
    alt = 0.5 - vv
    rgb = np.where(alt[..., None] >= 0, 0.2 + 0.3 * (1.0 - 2.0 * alt[..., None]) * np.array([1.0, 0.95, 0.85]),
                   np.array([0.04, 0.035, 0.03]))
    theta, phi = vv * math.pi, (uu - 0.5) * 2.0 * math.pi
    d = np.stack([np.sin(theta) * np.sin(phi), np.cos(theta), -np.sin(theta) * np.cos(phi)], -1)
    st, sp = math.radians(90.0 - sun_altitude_deg), (sun_u - 0.5) * 2.0 * math.pi
    s = np.array([math.sin(st) * math.sin(sp), math.cos(st), -math.sin(st) * math.cos(sp)])
    rgb[(d @ s) >= math.cos(math.radians(0.25))] = sun_radiance * np.array([1.0, 0.96, 0.9])
    out = np.ones((height, width, 4), np.float32)
    out[..., :3] = rgb
    return out


def env_sunlit(width=320, height=180, mode=MODE_IMAGE, denoise=True, ref_depth=1, sky_width=2048, sky_height=1024):
    """Exercises environment-map sampling (ST_OPT_ENVIRONMENT_MAP_SAMPLING): a ground plane and one occluder (a wall that casts the
    sun's shadow), no lights, lit only by sunlit_sky (the analytic sun is below the horizon).  The camera is still."""
    materials = {140: (material((0.6, 0.58, 0.55, 1.0)), False), 141: (material((0.7, 0.45, 0.3, 1.0), perceptual_roughness=0.5), False)}
    meshes = {240: np.stack(_quad((-30, 0, -30), (30, 0, -30), (30, 0, 30), (-30, 0, 30), (0, 1, 0))),
              241: np.stack(_box((-1.5, 0.0, -1.2), (1.5, 1.6, -0.9)))}
    instances = [(340, 240, 140, IDENTITY_AFFINE), (341, 241, 141, IDENTITY_AFFINE)]
    cam = dict(mode=mode, denoise=denoise, ref_depth=ref_depth, w=width, h=height, transform=look_at_transform((0.0, 2.2, 4.5), (0.0, 0.3, -0.5)),
               projection=perspective_infinite_reverse_rh(math.pi / 3.0, width / height, 0.1))
    return dict(name="env_sunlit", meshes=meshes, materials=materials, instances=instances, lights=[], sun=(0.0, -1.2), camera=cam,
                environment_map=dict(rgba=sunlit_sky(sky_width, sky_height), intensity=1.0, rotation=0.0))
