"""Float64 restatement of the normal-mapping rule (ST_OPT_NORMAL_MAPS, DESIGN.md §2 "Normal maps"), vectorised numpy.

Input: the baked triangle stream, the material table, the normal-map images of the scene, the camera uniform and the primary-hit
triangle of every pixel (prim_triangle_ids).  The barycentrics are rebuilt in float64 from the camera ray (camera.rs:80-93) and the
hit triangle (Möller–Trumbore, triangle.rs:64-113); the rule is then evaluated in float64:

    N  = normalize(u n1 + v n2 + (1 - u - v) n0)
    T4 = u t1 + v t2 + (1 - u - v) t0          T = T4.xyz (not renormalised), w = T4.w
    B  = w (N x T)
    Nt = 2 byte / 255 - 1                        (nearest texel of the repeat-wrapped uv, linear decode)
    n' = normalize((Nt.x T + Nt.y B) + Nt.z N); n' = N where n' is not finite or n'.N <= 0
    normal = n' copysign(1, inv_det)

Every pixel gets a derived error bound for a float32 evaluation of the same rule (what the kernels do) read back through the
octahedral surface map.  Two decisions are discrete: the nearest texel (a uv on a texel edge) and the n'.N > 0 test; where the
float64 margin of such a decision is inside the bound, the other outcome is computed too and either is accepted (and counted).

`evaluate(..., dtype=np.float32, mutation=...)` evaluates the rule in float32 numpy instead (one IEEE rounding per operation, in
the kernels' order), optionally with one deliberate mistake: the tests use it to show that the bound separates the rule from each
of those mistakes.
"""
import numpy as np

ATLAS = 8192
EPS32 = 2.0 ** -24
MUTATIONS = ("srgb_decode", "cross_order", "no_backface_sign", "renormalise_tangent", "no_fallback")


def srgb_to_linear(c):
    c = np.asarray(c, np.float64)
    return np.where(c <= 0.04045, c / 12.92, ((c + 0.055) / 1.055) ** 2.4)


def oct_decode(e):
    """normal.rs:23-34 in float64."""
    e = np.asarray(e, np.float64)
    m = e * 2.0 - 1.0
    n = np.stack([m[..., 0], m[..., 1], 1.0 - np.abs(m[..., 0]) - np.abs(m[..., 1])], axis=-1)
    t = np.maximum(-n[..., 2], 0.0)
    n[..., 0] -= np.copysign(t, n[..., 0])
    n[..., 1] -= np.copysign(t, n[..., 1])
    with np.errstate(invalid="ignore", divide="ignore"):
        return n / np.linalg.norm(n, axis=-1, keepdims=True)


def camera_rays(cam40, w, h):
    """Camera::ray (camera.rs:80-93) in float64 for every pixel: origins and unit directions, (h, w, 3) each."""
    c = np.asarray(cam40, np.float64).reshape(-1)
    n2w = c[16:32].reshape(4, 4)   # columns
    py, px = np.mgrid[0:h, 0:w].astype(np.float64)
    ndc_x = (px + 0.5) * 2.0 / c[36] - 1.0
    ndc_y = -((py + 0.5) * 2.0 / c[37] - 1.0)

    def project(z):
        p = np.stack([ndc_x, ndc_y, np.full_like(ndc_x, z), np.ones_like(ndc_x)], axis=-1)
        q = p @ n2w   # sum_k p[k] * column k
        return q[..., :3] / q[..., 3:4]
    far, near = project(float(np.float32(1.1920929e-07))), project(1.0)
    d = far - near
    return near, d / np.linalg.norm(d, axis=-1, keepdims=True)


def material_of_triangles(bvh, n_tri):
    """Material id per triangle from the BVH stream (serializer.rs:53-104): internal nodes are four float4 with d0.w = 0, leaf
    entries one float4 (flags, triangle id, material id, non-zero)."""
    e = np.asarray(bvh, np.float32).reshape(-1, 4).view(np.uint32)
    mat = np.full(n_tri, 0xffffffff, np.uint32)
    ptr = 0
    while ptr < len(e):
        if e[ptr, 3] == 0:
            ptr += 4
        else:
            mat[e[ptr, 1]] = e[ptr, 2]
            ptr += 1
    return mat


def _wrap(t):   # Material::sample_atlas's repeat wrap (material.rs:76-104)
    return np.where(t > 0.0, np.fmod(t, 1.0), 1.0 - np.fmod(-t, 1.0))


def evaluate(triangles, mat_tri, materials, images_by_rect, cam40, tid, w, h, dtype=np.float64, mutation=None):
    """The rule for every pixel whose primary hit is a triangle.  `mat_tri`: material id per triangle (material_of_triangles);
    `images_by_rect`: {(x, y, w, h) texel rect in the atlas: RGBA8
    image}.  Returns a dict of (h, w, ...) arrays: `normal` (the shading normal; NaN where nothing was hit), `bound`, `alt` (the
    other outcome of a discrete decision inside its margin, NaN elsewhere), `unknown` (the uv sits on the edge of the image's
    rect: the other texel belongs to a neighbour in the atlas), `mapped` (the material has a normal map), `fallback`
    (n' was replaced by N), `material`."""
    assert mutation in (None,) + MUTATIONS
    tri = np.asarray(triangles, np.float32).reshape(-1, 9, 4)
    mats = np.asarray(materials, np.float32).reshape(-1, 28)
    tid = np.asarray(tid).reshape(h, w).view(np.uint32)
    hit = tid != 0xffffffff
    idx = np.where(hit, tid, 0).astype(np.int64)
    T = tri[idx].astype(np.float64)                       # (h, w, 9, 4)
    p0, p1, p2 = T[..., 0, :3], T[..., 3, :3], T[..., 6, :3]
    o, d = camera_rays(cam40, w, h)
    e1, e2 = p1 - p0, p2 - p0
    pvec = np.cross(d, e2)
    det = np.einsum("...k,...k", e1, pvec)
    with np.errstate(divide="ignore", invalid="ignore"):
        inv_det = 1.0 / det
        tvec = o - p0
        u = np.einsum("...k,...k", tvec, pvec) * inv_det
        qvec = np.cross(tvec, e1)
        v = np.einsum("...k,...k", d, qvec) * inv_det
        t_hit = np.einsum("...k,...k", e2, qvec) * inv_det
    n0, n1, n2 = T[..., 1, :3], T[..., 4, :3], T[..., 7, :3]
    t0, t1, t2 = T[..., 2, :], T[..., 5, :], T[..., 8, :]
    uv0, uv1, uv2 = T[..., [0, 1], 3], T[..., [3, 4], 3], T[..., [6, 7], 3]
    sign = np.copysign(1.0, inv_det)

    # barycentric uncertainty of the kernels' float32 hit: the float32 camera ray and Möller–Trumbore carry a few ulps of relative
    # error in (origin, direction, edge vectors); a ray error of eps_r moves the hit by eps_r (|o| + t) across the triangle, i.e.
    # the barycentrics by that over the triangle's smallest altitude.
    area2 = np.linalg.norm(np.cross(e1, e2), axis=-1)
    longest = np.maximum(np.maximum(np.linalg.norm(e1, axis=-1), np.linalg.norm(e2, axis=-1)), np.linalg.norm(p2 - p1, axis=-1))
    with np.errstate(divide="ignore", invalid="ignore"):
        dbary = 64.0 * EPS32 * (np.linalg.norm(o, axis=-1) + np.abs(t_hit) + np.linalg.norm(p0, axis=-1)) * longest / area2 + 16.0 * EPS32

    f = dtype
    if dtype is np.float32:   # the kernels' order of operations, one float32 rounding per operation
        uu, vv = u.astype(f), v.astype(f)
    else:
        uu, vv = u, v
    ww = (f(1.0) - uu) - vv

    def mix(a0, a1, a2):
        a0, a1, a2 = a0.astype(f), a1.astype(f), a2.astype(f)
        return (a1 * uu[..., None] + a2 * vv[..., None]) + a0 * ww[..., None]

    def norm(a):
        with np.errstate(divide="ignore", invalid="ignore"):
            return a * (f(1.0) / np.sqrt(np.einsum("...k,...k", a, a)))[..., None]

    def cross(a, b):   # glam's Vec3::cross, component order as xcross
        return np.stack([a[..., 1] * b[..., 2] - b[..., 1] * a[..., 2], a[..., 2] * b[..., 0] - b[..., 2] * a[..., 0],
                         a[..., 0] * b[..., 1] - b[..., 0] * a[..., 1]], axis=-1)

    N = norm(mix(n0, n1, n2))
    T4 = mix(t0, t1, t2)
    Tv = T4[..., :3]
    if mutation == "renormalise_tangent":
        Tv = norm(Tv)
    B = (cross(Tv, N) if mutation == "cross_order" else cross(N, Tv)) * T4[..., 3:4]
    uv = mix(np.concatenate([uv0, np.zeros_like(uv0[..., :1])], -1), np.concatenate([uv1, np.zeros_like(uv1[..., :1])], -1),
             np.concatenate([uv2, np.zeros_like(uv2[..., :1])], -1))[..., :2].astype(np.float64)

    # uv uncertainty of the kernels' float32 uv: the barycentric uncertainty times the uv spread of the triangle, plus the
    # roundings of the float32 interpolation (three products and two sums of terms below |uv| + spread) and of the wrap / rect
    # mapping (two more); in texels it is this times the image size
    uv_spread = np.maximum(np.maximum(np.abs(uv1 - uv0), np.abs(uv2 - uv0)), np.abs(uv2 - uv1))
    duv = uv_spread * dbary[..., None] * 2.0 + 8.0 * EPS32 * (np.abs(uv) + uv_spread + 1.0)

    mat = np.full((h, w), 0xffffffff, np.uint32)
    out = dict(material=mat)
    rect = np.zeros((h, w, 4))
    mat[hit] = mat_tri[tid[hit]]
    rect[hit] = mats[mat_tri[tid[hit]], 24:28]
    mapped = hit & np.any(rect != 0, axis=-1)
    rect_tx = np.round(rect * ATLAS).astype(np.int64)   # texel rect (exact: the rect is a multiple of 1 / 8192)

    # nearest texel (+ the neighbour across the edge where the coordinate is within the margin)
    texel = np.zeros((h, w, 3))
    alt_texel = np.full((h, w, 3), np.nan)
    unknown = np.zeros((h, w), bool)
    for key, img in images_by_rect.items():
        sel = mapped & np.all(rect_tx == np.asarray(key), axis=-1)
        if not sel.any():
            continue
        ih, iw = img.shape[:2]
        dec = srgb_to_linear(img[..., :3] / 255.0) if mutation == "srgb_decode" else img[..., :3].astype(np.float64) / 255.0
        cs = np.stack([_wrap(uv[sel][:, 0]) * iw, _wrap(uv[sel][:, 1]) * ih], axis=-1)
        ix = np.floor(cs).astype(np.int64)
        near_edge = np.abs(cs - np.round(cs)) <= duv[sel] * np.array([iw, ih])
        other = np.where(cs - ix >= 0.5, ix + 1, ix - 1)
        lim = np.array([iw, ih])
        inside = (ix >= 0) & (ix < lim)
        unknown_sel = np.any(~inside, axis=-1) | np.any(near_edge & ((other < 0) | (other >= lim)), axis=-1)
        ixc = np.clip(ix, 0, lim - 1)
        texel[sel] = dec[ixc[:, 1], ixc[:, 0]]
        amb = np.any(near_edge, axis=-1) & ~unknown_sel
        if amb.any():
            ox = np.where(near_edge, np.clip(other, 0, lim - 1), ixc)
            a = alt_texel[sel]
            a[amb] = dec[ox[amb, 1], ox[amb, 0]]
            alt_texel[sel] = a
        unknown[sel] = unknown_sel

    def apply(tex):
        nt = (f(2.0) * tex.astype(f) - f(1.0))
        M = (Tv * nt[..., 0:1] + B * nt[..., 1:2]) + N * nt[..., 2:3]
        m = norm(M)
        with np.errstate(invalid="ignore"):
            dot = np.einsum("...k,...k", m, N)
            ok = np.all(np.isfinite(m), axis=-1) & (dot > 0)
        if mutation == "no_fallback":
            ok = np.ones_like(ok)
        return np.where(ok[..., None], m, N), ok, M, dot

    mapped_n, ok, M, dot = apply(texel)
    n = np.where(mapped[..., None], mapped_n, N)
    if mutation != "no_backface_sign":
        n = n * sign[..., None]

    # ---- the bound (float64 only) ----
    n64 = n.astype(np.float64)
    spread = lambda a0, a1, a2: np.maximum(np.maximum(np.linalg.norm(a1 - a0, axis=-1), np.linalg.norm(a2 - a0, axis=-1)), np.linalg.norm(a2 - a1, axis=-1))
    dN = spread(n0, n1, n2) * dbary * 2.0 / np.maximum(np.linalg.norm(u[..., None] * n1 + v[..., None] * n2 + (1 - u - v)[..., None] * n0, axis=-1), 1e-3) + 8 * EPS32
    dT = spread(t0[..., :3], t1[..., :3], t2[..., :3]) * dbary * 2.0 + 8 * EPS32
    dw = spread(t0[..., 3:], t1[..., 3:], t2[..., 3:]) * dbary * 2.0 + 4 * EPS32
    Tn = np.linalg.norm(Tv.astype(np.float64), axis=-1)
    nt64 = 2.0 * texel - 1.0
    dB = np.abs(T4[..., 3].astype(np.float64)) * (dN * Tn + dT + 4 * EPS32 * Tn) + dw * Tn
    Bn = np.linalg.norm(B.astype(np.float64), axis=-1)
    Mabs = np.abs(nt64[..., 0]) * Tn + np.abs(nt64[..., 1]) * Bn + np.abs(nt64[..., 2])
    dM = np.abs(nt64[..., 0]) * dT + np.abs(nt64[..., 1]) * dB + np.abs(nt64[..., 2]) * dN + 12 * EPS32 * Mabs
    with np.errstate(divide="ignore", invalid="ignore"):
        Mn = np.linalg.norm(M.astype(np.float64), axis=-1)
        dmapped = 2.0 * dM / Mn + 8 * EPS32
    oct_err = 16 * EPS32   # octahedral encode (float32) + decode of the surface map
    bound = np.where(mapped & ok, dmapped, dN) + oct_err

    alt = np.full((h, w, 3), np.nan)
    # n'.N > 0 decided inside the margin: the other outcome is acceptable too
    margin_fb = mapped & np.isfinite(dot) & (np.abs(dot) <= bound)
    alt[margin_fb] = np.where(ok[margin_fb][:, None], N[margin_fb], mapped_n[margin_fb]) * sign[margin_fb][:, None]
    amb_tex = mapped & np.isfinite(alt_texel[..., 0]) & ~margin_fb
    if amb_tex.any():
        an, _, _, _ = apply(np.where(np.isfinite(alt_texel), alt_texel, texel))
        alt[amb_tex] = an[amb_tex] * sign[amb_tex][:, None]
    n64[~hit] = np.nan
    out.update(normal=n64, bound=bound, alt=alt, unknown=unknown & mapped, mapped=mapped, fallback=mapped & ~ok, hit=hit,
               margin_texel=amb_tex, margin_fallback=margin_fb, sign=sign)
    return out


def images_by_rect(materials, scene):
    """{texel rect: image} for the normal maps of `scene`, matched to the uploaded material rects by size."""
    mats = np.asarray(materials, np.float32).reshape(-1, 28)
    rects = {tuple(np.round(r * ATLAS).astype(np.int64)) for r in mats[:, 24:28] if np.any(r != 0)}
    handles = {tex["normal_map"] for tex in scene.get("material_textures", {}).values() if tex.get("normal_map") is not None}
    out = {}
    for r in rects:
        match = [hd for hd in handles if scene["images"][hd].shape[1] == r[2] and scene["images"][hd].shape[0] == r[3]]
        assert len(match) == 1, f"normal map of rect {r} is not identified by its size"
        out[r] = scene["images"][match[0]]
    return out


def check(got, ref, skip=None):
    """Device normals `got` (h, w, 3) against the restatement: inside the bound of `normal`, or of `alt` where a discrete decision
    sits inside its margin.  Returns counts; raises with the first offenders."""
    got = np.asarray(got, np.float64)
    hit = ref["hit"] & ~ref["unknown"]
    if skip is not None:
        hit &= ~skip
    err = np.linalg.norm(got - ref["normal"], axis=-1)
    err_alt = np.linalg.norm(got - np.where(np.isfinite(ref["alt"]), ref["alt"], np.inf), axis=-1)
    with np.errstate(invalid="ignore"):
        good = (err <= ref["bound"]) | (err_alt <= ref["bound"])
    bad = hit & ~good
    took_alt = hit & (err_alt <= ref["bound"]) & ~(err <= ref["bound"])
    if bad.any():
        ys, xs = np.nonzero(bad)
        k = list(zip(ys[:5].tolist(), xs[:5].tolist()))
        raise AssertionError(f"{int(bad.sum())}/{int(hit.sum())} normals outside the float64 bound; first at (y, x) {k}: got "
                             f"{got[bad][:3].tolist()} want {ref['normal'][bad][:3].tolist()} bound {ref['bound'][bad][:3].tolist()}")
    with np.errstate(invalid="ignore"):
        worst = float(np.nanmax(np.where(hit, np.minimum(err, err_alt) / ref["bound"], 0.0)))
    return dict(pixels=int(hit.sum()), mapped=int((hit & ref["mapped"]).sum()), fallback=int((hit & ref["fallback"]).sum()),
                texel_margin=int((hit & ref["margin_texel"]).sum()), fallback_margin=int((hit & ref["margin_fallback"]).sum()),
                took_alt=int(took_alt.sum()), unknown=int(ref["unknown"].sum()), worst_ratio=worst)
