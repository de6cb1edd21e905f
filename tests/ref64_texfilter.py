"""Float64 restatement of ST_OPT_TEXTURE_FILTER's fetch (DESIGN.md §2 "Texture filtering") with a derived error bound.

Written from the rule, not from the CUDA or oracle code: the mip chains, the ray-cone level of detail and the trilinear sample with
repeat-wrapped taps.  Its inputs are what the rule takes from the rest of the renderer, as float32 values: the triangle (positions,
uvs), the hit uv, the ray direction, the hit distance and the camera rays of the pixel and of its right and lower neighbours
(`oracle_texfilter` exports them per hit with the filtered results it computed, `TextureFilterOracleEngine.probe`).

The bound covers the float32 evaluation of the rule, term by term (u = 2^-24 is the unit roundoff):
- cone width: the differences of the camera rays are rounded once (u relative), t (d1 - d0) and the sum once more each, the length
  3u: |dw| <= |dv| + 3u w with |dv_i| <= 4u (|o1_i - o0_i| + |t| |d1_i - d0_i|);
- q = A_uv W H w^2 |c| / (c.d)^2: the edge and uv differences (u each), the products and sums of the cross products (<= 5u of the sum
  of the magnitudes of their terms), |c| (3u), c.d (3u of the sum of |c_i d_i| plus the propagated error of c), the five products
  and the division (6u): a relative bound rho on q;
- lambda = 0.5 log2 q: 0.5 rho / ln 2, plus log2_x's own bound 2^-21 (1 + |log2 q|) / 2;
- texel coordinate s = u w_k - 0.5: the wrap (u), the product and the difference (2u of the magnitudes);
- the bilinear and level blends: the weights' errors times the differences of the blended texels, plus 8u per blend.
First-order terms only; the bound is doubled to cover the second-order ones.

A level or a texel choice is compared only where lambda, or the texel coordinate, is farther than its bound from the decision edge
(an integer); the other hits are counted as undecided.
"""
import math

import numpy as np

U = 2.0 ** -24
ATLAS = 8192.0
PROBE_WORDS = 40


def numpy_level(img, lut, mid):
    """Level k + 1 of `img` (h, w, 4) uint8: the 2x2 box (edge texels repeated) averaged through the sRGB table in float32 as the rule
    orders it, re-encoded to the byte whose table value is nearest (ties to the lower byte); alpha averaged on the bytes."""
    h, w = img.shape[:2]
    nw, nh = max(1, w >> 1), max(1, h >> 1)
    xs = np.arange(nw); ys = np.arange(nh)
    xa, xb = np.minimum(2 * xs, w - 1), np.minimum(2 * xs + 1, w - 1)
    ya, yb = np.minimum(2 * ys, h - 1), np.minimum(2 * ys + 1, h - 1)
    c00, c10 = img[ya][:, xa], img[ya][:, xb]
    c01, c11 = img[yb][:, xa], img[yb][:, xb]
    out = np.empty((nh, nw, 4), np.uint8)
    for ch in range(3):
        s = (((lut[c00[..., ch]] + lut[c10[..., ch]]).astype(np.float32) + lut[c01[..., ch]]).astype(np.float32) + lut[c11[..., ch]]).astype(np.float32)
        s = (s * np.float32(0.25)).astype(np.float32)
        out[..., ch] = np.searchsorted(mid, s, side="left")   # the count of midpoints strictly below: ties go to the lower byte
    out[..., 3] = ((c00[..., 3].astype(np.uint32) + c10[..., 3] + c01[..., 3] + c11[..., 3] + 2) >> 2).astype(np.uint8)
    return out


def mip_chain(img, lut):
    """[level 0, level 1, ...] of `img` as uint8 arrays."""
    lut = np.asarray(lut, np.float32)
    mid = ((lut[:-1] + lut[1:]).astype(np.float32) * np.float32(0.5)).astype(np.float32)
    levels = [np.asarray(img, np.uint8)]
    while levels[-1].shape[0] > 1 or levels[-1].shape[1] > 1:
        levels.append(numpy_level(levels[-1], lut, mid))
    return levels


def atlas_rects(scene):
    """{texel rect (x, y, w, h): handle}: the shelf placement st_insert_image gives the scene's images in insertion order."""
    x = y = shelf_h = 0
    out = {}
    for hnd, img in scene["images"].items():
        h, w = img.shape[:2]
        if x + w > ATLAS:
            x, y, shelf_h = 0, y + shelf_h, 0
        out[(x, y, w, h)] = hnd
        x += w; shelf_h = max(shelf_h, h)
    return out


class Restatement:
    def __init__(self, scene, triangles, materials, lut):
        self.tri = np.asarray(triangles, np.float32).reshape(-1, 9, 4).astype(np.float64)
        self.mats = np.asarray(materials, np.float32).reshape(-1, 28).astype(np.float64)
        self.lut = np.asarray(lut, np.float32).astype(np.float64)
        self.rects = atlas_rects(scene)
        self.chains = {}
        for r, hnd in self.rects.items():
            self.chains[r] = [self._decode(l) for l in mip_chain(scene["images"][hnd], lut)]

    def _decode(self, level):
        d = np.empty(level.shape, np.float64)
        d[..., :3] = self.lut[level[..., :3]]
        d[..., 3] = level[..., 3] / 255.0
        return d

    def slot(self, mid, k):
        """(rect as texels or None, factor) of material `mid`'s slot k (0 base colour, 1 emissive, 2 metallic-roughness)."""
        m = self.mats[mid]
        rect = m[[4, 12, 20][k]:[4, 12, 20][k] + 4]
        factor = [m[0:4], m[8:12], np.array([1.0, m[16], m[17], 1.0])][k]
        if not rect.any():
            return None, factor
        return tuple(int(v) for v in np.round(rect * ATLAS)), factor

    def lod(self, rec, W, H, L):
        """(lambda, its bound) of a probe record for a W x H image of L levels; bound None = degenerate (no decision possible)."""
        t = self.tri[int(np.float32(rec[1]).view(np.uint32))]
        p0, p1, p2 = t[0, :3], t[3, :3], t[6, :3]
        e1, e2 = p1 - p0, p2 - p0
        c = np.cross(e1, e2)
        cabs = np.array([abs(e1[1] * e2[2]) + abs(e1[2] * e2[1]), abs(e1[2] * e2[0]) + abs(e1[0] * e2[2]), abs(e1[0] * e2[1]) + abs(e1[1] * e2[0])])
        dc = 5 * U * cabs
        clen = float(np.linalg.norm(c))
        dclen = float(np.linalg.norm(dc)) + 3 * U * clen
        d = rec[5:8].astype(np.float64)
        cd = float(c @ d)
        dcd = float(np.abs(dc) @ np.abs(d)) + 3 * U * float(np.abs(c * d).sum())
        du1, dv1, du2, dv2 = t[3, 3] - t[0, 3], t[4, 3] - t[1, 3], t[6, 3] - t[0, 3], t[7, 3] - t[1, 3]
        area = abs(du1 * dv2 - du2 * dv1)
        darea = 5 * U * (abs(du1 * dv2) + abs(du2 * dv1))
        tt = float(rec[8])
        o = [rec[10 + 6 * k:13 + 6 * k].astype(np.float64) for k in range(3)]
        dr = [rec[13 + 6 * k:16 + 6 * k].astype(np.float64) for k in range(3)]
        if rec[9] > 0.5:
            vs = [(o[k] - o[0]) + tt * (dr[k] - dr[0]) for k in (1, 2)]
            dvs = [4 * U * (np.abs(o[k] - o[0]) + abs(tt) * np.abs(dr[k] - dr[0])) for k in (1, 2)]
            lens = [float(np.linalg.norm(v)) for v in vs]
            w = max(lens)
            dw = max(float(np.linalg.norm(dv)) for dv in dvs) + 3 * U * w
        else:
            dd = [dr[k] - dr[0] for k in (1, 2)]
            m = max(float(np.linalg.norm(x)) for x in dd)
            w = tt * m
            dw = abs(tt) * (max(float(np.linalg.norm(U * np.abs(x))) for x in dd) + 3 * U * m) + U * abs(w)
        top = float(L - 1)
        if area == 0.0 or cd == 0.0 or w == 0.0 or clen == 0.0:
            return (0.0 if area == 0.0 or w == 0.0 or clen == 0.0 else top), None
        rho = darea / area + 2 * dw / abs(w) + dclen / clen + 2 * dcd / abs(cd) + 6 * U
        if rho > 0.05 or darea >= area:
            return None, None
        q = area * W * H * w * w * clen / (cd * cd)
        lam = 0.5 * math.log2(q)
        dlam = 2.0 * (0.5 * rho / math.log(2.0) + 0.5 * 2.0 ** -21 * (1.0 + abs(math.log2(q))) + 2 * U * abs(lam))
        return lam, dlam

    def _bilinear(self, lvl, uu, vv):
        """float64 bilinear on decoded level `lvl` at wrapped (u, v); returns value, bound, and decided (texel choice clear)."""
        h, w = lvl.shape[:2]
        s, t = uu * w - 0.5, vv * h - 0.5
        ds = 2 * (w * U + 2 * U * (abs(uu * w) + 0.5))
        dt = 2 * (h * U + 2 * U * (abs(vv * h) + 0.5))
        fs, ft = s - math.floor(s), t - math.floor(t)
        decided = min(fs, 1 - fs) > ds and min(ft, 1 - ft) > dt
        x0, y0 = int(math.floor(s)), int(math.floor(t))
        xa, xb, ya, yb = x0 % w, (x0 + 1) % w, y0 % h, (y0 + 1) % h
        c00, c10, c01, c11 = lvl[ya, xa], lvl[ya, xb], lvl[yb, xa], lvl[yb, xb]
        val = (c00 * (1 - fs) + c10 * fs) * (1 - ft) + (c01 * (1 - fs) + c11 * fs) * ft
        dx = np.maximum(np.abs(c10 - c00), np.abs(c11 - c01))
        dy = np.maximum(np.abs(c01 - c00), np.abs(c11 - c10))
        return val, 2 * (ds * dx + dt * dy + 8 * U), decided

    def sample(self, rec, k):
        """(value (4,), bound (4,)) of slot k at probe record `rec`, or None where a level or texel choice is undecided."""
        rect, factor = self.slot(int(np.float32(rec[2]).view(np.uint32)), k)
        if rect is None:
            return factor, np.zeros(4)
        lv = self.chains.get(rect)
        assert lv is not None, f"no image at rect {rect}"
        W, H = rect[2], rect[3]
        wrap = lambda x: math.fmod(x, 1.0) if x > 0 else 1.0 - math.fmod(-x, 1.0)
        uu, vv = wrap(float(rec[3])), wrap(float(rec[4]))
        L = len(lv)
        lam, dlam = (0.0, 0.0) if L == 1 else self.lod(rec, W, H, L)
        if lam is None:
            return None
        if dlam is None:
            dlam = 0.0
        if dlam > 0 and any(abs(lam - j) <= dlam for j in range(L)):
            return None   # the level choice (or the clamp to [0, levels - 1]) is within the bound of its edge
        lam = min(max(lam, 0.0), float(L - 1))
        k0 = int(math.floor(lam)); fl = lam - k0
        v0, b0, ok0 = self._bilinear(lv[k0], uu, vv)
        if not ok0:
            return None
        val, bnd = v0, b0
        if fl > 0 and k0 + 1 < L:
            v1, b1, ok1 = self._bilinear(lv[k0 + 1], uu, vv)
            if not ok1:
                return None
            val = v0 * (1 - fl) + v1 * fl
            bnd = np.maximum(b0, b1) + 2 * (dlam * np.abs(v1 - v0) + 4 * U)
        return factor * val, np.abs(factor) * bnd + 2 * U * np.abs(factor * val) + 1e-30


def check(rest, records, slots=(0, 1, 2)):
    """Compares every valid probe record's filtered terms with the restatement.  Raises AssertionError ("outside the float64 bound")
    if a decided term leaves its bound; returns the counts (hits, checked terms, undecided terms, worst error / bound)."""
    stats = dict(hits=0, checked=0, undecided=0, worst_ratio=0.0, outside=0)
    for rec in records[records[:, 0] == 1.0]:
        stats["hits"] += 1
        for k in slots:
            r = rest.sample(rec, k)
            if r is None:
                stats["undecided"] += 1
                continue
            want, bound = r
            got = rec[[28, 32, 36][k]:[28, 32, 36][k] + 4].astype(np.float64)
            n = 3 if k == 1 else 4   # emissive has no alpha
            err = np.abs(got[:n] - want[:n])
            stats["checked"] += 1
            ratio = float(np.max(np.where(bound[:n] > 0, err / np.maximum(bound[:n], 1e-300), np.where(err > 0, np.inf, 0.0))))
            stats["worst_ratio"] = max(stats["worst_ratio"], ratio)
            if ratio > 1.0:
                stats["outside"] += 1
    if stats["outside"]:
        raise AssertionError(f"{stats['outside']} terms outside the float64 bound: {stats}")
    return stats
