"""Float64 restatement of depth of field (ST_OPT_DEPTH_OF_FIELD; DESIGN.md §2 "Depth of field"), with derived bounds on the f32
evaluation.

Inputs taken as they are: the f32 `output`, the f32 hit distances t, the f32 camera ray directions d, and the lens constants (the rule
rounds each to f32 once, from double: restated here in double and rounded the same way).  u = 2^-24.
- CoC: z = t (d . fwd) within u |z| + 3 u t sum |d_i fwd_i| (two products, two additions, one product); g = (z - F) / z moves by
  (F / z) |dz| / z for dz, plus one rounding of z - F (u |z - F| / z) and one of the quotient (u |g|); r = k g adds u |r| (the product
  is taken before the quotient in f32; the same two roundings).  The clamp to [-R, R] does not widen the bound, and where both ends
  of the bound clamp, r is exactly +-R.  The sky's r = min(k, R)
  is exact.
- Tiles: M, the max of |r| over the tile's neighbourhood, lies in [max(|r| - dr), max(|r| + dr)].  rho = 0 when M < 1/2, ceil(M)
  otherwise: a tile whose interval gives two different rho is undecided, and so is each of its pixels.
- Gather: s = (r_q > r_p) ? min(|r_q|, |r_p|) : |r_q| is continuous in (r_q, r_p) (at r_q = r_p both branches give |r_q|), so it moves by
  at most dr_q + dr_p: no depth comparison needs deciding.  w = clamp(s - delta + 1, 0, 1) / max(s, 1/2)^2 is Lipschitz in s with
  constant 1 / m^2 + 2 / m^3 (m = max(s - ds, 1/2)), plus u per rounding.  The sums N = sum w c and D = sum w over n = 81 taps carry
  (n + 1) u of their absolute sums; x = N / D moves by (dN + |x| dD) / D plus u |x|.
Every bound is doubled for the second-order terms.  A copied tile (rho = 0) is checked bit for bit.
"""
import math

import numpy as np

U = 2.0 ** -24
TILE, MAX_RADIUS, TAPS, HEADER = 16, 32, 81, 16


def _round_half_away(v):
    return -math.floor(-v + 0.5) if v < 0 else math.floor(v + 0.5)


def taps():
    """The tap table, restated: (32 x 81 x 2) offsets, (32 x 81) distances (float32)."""
    dxy = np.zeros((MAX_RADIUS, TAPS, 2), np.int64)
    d = np.zeros((MAX_RADIUS, TAPS), np.float32)
    for rho in range(1, MAX_RADIUS + 1):
        i = 1
        for j in range(1, 5):
            for a_i in range(8 * j):
                a, rad = 2.0 * math.pi * a_i / (8 * j), rho * j / 4.0
                dx, dy = _round_half_away(rad * math.cos(a)), _round_half_away(rad * math.sin(a))
                dxy[rho - 1, i] = (dx, dy)
                d[rho - 1, i] = np.float32(math.sqrt(dx * dx + dy * dy))
                i += 1
    return dxy, d


def consts(p, transform16, projection16, h):
    """(defocused, {f, A, k, F, R, fwd (3)} as float32), in double from the f32 settings, each rounded once."""
    f32 = lambda v: float(np.float32(v))
    sh, N, F = f32(p["sensor_height"]), f32(p["aperture_f_stops"]), f32(p["focal_distance"])
    t = np.asarray(transform16, np.float32).astype(np.float64)
    f = 0.5 * sh * float(np.float32(projection16[5]))
    A = f / N
    active = F > f
    k = A * f / (F - f) * h / sh / 2.0 if active else 0.0
    fw = -t[8:11]
    fw = fw / math.sqrt(float((fw * fw).sum()))
    return active, np.array([f, A, k, F, f32(p["max_radius"]), fw[0], fw[1], fw[2]], np.float32)


def coc(t, d, c, active):
    """r (float64) and its bound, per pixel (t: h x w, d: h x w x 3 float32 inputs)."""
    k, F, R = (float(v) for v in c[2:5])
    fw = c[5:8].astype(np.float64)
    t = np.asarray(t, np.float32).astype(np.float64)
    d = np.asarray(d, np.float32).astype(np.float64)
    if not active:
        return np.zeros_like(t), np.zeros_like(t)
    dot = (d * fw).sum(-1)
    z = t * dot
    dz = U * np.abs(z) + 3 * U * t * np.abs(d * fw).sum(-1)
    with np.errstate(divide="ignore", invalid="ignore"):
        g = (z - F) / z
        dg = (F / np.abs(z)) * dz / np.abs(z) + U * np.abs(z - F) / np.abs(z) + U * np.abs(g)
    r = k * g
    dr = abs(k) * dg + 2 * U * np.abs(r)
    dr = np.where(np.abs(r) - 2 * dr >= R, 0.0, dr)   # clamped however the f32 rounds: exactly +-R
    r = np.clip(r, -R, R)
    sky = t == 0
    r = np.where(sky, min(k, R), r)
    dr = np.where(sky, 0.0, dr)
    return r, 2.0 * dr


def _rho(M):
    return np.where(M < 0.5, 0, np.ceil(M)).astype(np.int64)


def tiles(r, dr, R):
    """Per tile: rho (float64 decision), decided (every M in [max(|r| - dr), max(|r| + dr)] gives it)."""
    h, w = r.shape
    TX, TY = (w + TILE - 1) // TILE, (h + TILE - 1) // TILE
    a = np.abs(r)
    m, lo, hi = (np.zeros((TY, TX)) for _ in range(3))
    for ty in range(TY):
        for tx in range(TX):
            sl = (slice(ty * TILE, (ty + 1) * TILE), slice(tx * TILE, (tx + 1) * TILE))
            m[ty, tx], lo[ty, tx], hi[ty, tx] = a[sl].max(), (a[sl] - dr[sl]).max(), (a[sl] + dr[sl]).max()
    q = int(math.ceil(float(np.float32(R)) / TILE))
    M, Mlo, Mhi = (np.zeros_like(m) for _ in range(3))
    for ty in range(TY):
        for tx in range(TX):
            sl = (slice(max(0, ty - q), ty + q + 1), slice(max(0, tx - q), tx + q + 1))
            M[ty, tx], Mlo[ty, tx], Mhi[ty, tx] = m[sl].max(), lo[sl].max(), hi[sl].max()
    return _rho(M), _rho(Mlo) == _rho(Mhi)


def gather(output, r, dr, R):
    """The defocused frame in float64 with its bound, the per-pixel rho and decided mask (h x w)."""
    o = np.asarray(output, np.float32).reshape(r.shape + (4,))
    h, w = r.shape
    rho_t, dec_t = tiles(r, dr, R)
    rho = np.repeat(np.repeat(rho_t, TILE, 0), TILE, 1)[:h, :w]
    dec = np.repeat(np.repeat(dec_t, TILE, 0), TILE, 1)[:h, :w]
    c = np.where(np.isfinite(o[..., :3]), o[..., :3], np.float32(0)).astype(np.float64)
    x = o.astype(np.float64).copy()
    dx = np.zeros(r.shape + (3,))
    dxy, dist = taps()
    yy, xx = np.mgrid[0:h, 0:w]
    for g in np.unique(rho):
        if g == 0:
            continue
        sel = rho == g
        py, px = yy[sel], xx[sel]
        rp, drp = r[sel], dr[sel]
        N, D, aN, dN, dD = np.zeros((sel.sum(), 3)), np.zeros(sel.sum()), np.zeros((sel.sum(), 3)), np.zeros((sel.sum(), 3)), np.zeros(sel.sum())
        for i in range(TAPS):
            ddx, ddy = dxy[g - 1, i]
            qy, qx = np.clip(py + ddy, 0, h - 1), np.clip(px + ddx, 0, w - 1)
            rq, drq, cq = r[qy, qx], dr[qy, qx], c[qy, qx]
            s = np.where(rq > rp, np.minimum(np.abs(rq), np.abs(rp)), np.abs(rq))
            ds = drq + drp
            delta = float(dist[g - 1, i])
            cw = np.clip(s - delta + 1.0, 0.0, 1.0)
            m = np.maximum(s, 0.5)
            wt = cw / (m * m)
            mlo = np.maximum(s - ds, 0.5)
            dw = (1.0 / mlo ** 2 + 2.0 / mlo ** 3) * ds + U * (np.abs(s - delta) + np.abs(s - delta + 1.0)) / (m * m) + 3 * U * wt
            N += wt[:, None] * cq
            D += wt
            aN += wt[:, None] * np.abs(cq)
            dN += dw[:, None] * np.abs(cq)
            dD += dw
        dN += (TAPS + 1) * U * aN
        dD += (TAPS + 1) * U * D
        v = N / D[:, None]
        x[sel, :3] = v
        x[sel, 3] = 1.0
        dx[sel] = 2.0 * ((dN + np.abs(v) * dD[:, None]) / D[:, None] + U * np.abs(v))
    return x, dx, rho, dec


def check(words, frame, output, t, d, p, transform16, projection16, h, w):
    """Counts the words and frame values outside the float64 bound: the header, every r, every decided tile's rho, every decided pixel
    (bit for bit in a copied tile); returns (violations, undecided pixels)."""
    words = np.asarray(words, np.float32).reshape(-1)
    u = words.view(np.uint32)
    active, c = consts(p, transform16, projection16, h)
    TX, TY = (w + TILE - 1) // TILE, (h + TILE - 1) // TILE
    head = np.zeros(HEADER, np.uint32)
    head[:5] = (w, h, TX, TY, int(active))
    head[5:13] = c.view(np.uint32)
    bad = int((u[:HEADER] != head).sum())
    r32 = words[HEADER:HEADER + w * h].reshape(h, w).astype(np.float64)
    r, dr = coc(t, d, c, active)
    bad += int((~(np.abs(r32 - r) <= dr)).sum())   # a NaN is outside every bound
    x, dx, rho, dec = gather(output, r, dr, c[4])
    rho_t, dec_t = tiles(r, dr, c[4])
    got_rho = u[HEADER + w * h:HEADER + w * h + TX * TY].reshape(TY, TX).astype(np.int64)
    bad += int(((got_rho != rho_t) & dec_t).sum())
    f = np.asarray(frame, np.float32).reshape(h, w, 4)
    copied = dec & (rho == 0)
    o = np.asarray(output, np.float32).reshape(h, w, 4)
    bad += int((f[copied].view(np.uint32) != o[copied].view(np.uint32)).sum())
    blur = dec & (rho > 0)
    bad += int((~(np.abs(f[blur][:, :3].astype(np.float64) - x[blur][:, :3]) <= dx[blur])).sum()) + int((f[blur][:, 3] != 1.0).sum())
    return bad, int((~dec).sum())
