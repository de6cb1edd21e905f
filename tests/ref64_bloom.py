"""Float64 restatement of bloom (ST_OPT_BLOOM; DESIGN.md §2 "Bloom"), with derived bounds on the f32 evaluation.

Every texel carries (value, bound) per channel, the bound an absolute first-order bound on |f32 - float64|:
- Input: x = c s with s = 2^y within POW2_REL(y) (ref64_exposure), plus the multiply's rounding.  The prefilter's weight
  w = max(q, b - t) / max(b, 1e-4) is Lipschitz in b (clamp, square, max): its first-order term from b's bound, plus one rounding per
  operation.
- Down levels: the 13-tap filter is a weighted sum of non-negative terms with weights that sum to 1, so a level's bound is the same
  weighted sum of its inputs' bounds plus, per texel, 3 u of the value per chain of additions it went through (2 in the box, 2 in the
  group, 3 in the combination).  The Karis weights of the first level add their first-order term: the weighted average moves by at most
  sum |t_i - g| |dw_i| / sum w_i <= sum (t_i + g) |dw_i| / sum w_i, with dw_i = w_i^2 dL_i.
- Up levels: the tent (4 additions) and (1 - a) down + a tent (2 roundings), each the same non-negative combination of bounds.
- Store: x' = (1 - I) x + I B (mode 0) or x + I B (mode 1), then T through ref64_exposure.transform and the monotone sRGB store: a byte is
  decided where both ends of the interval give it.
Every bound is doubled for the second-order terms, as ref64_exposure does.
"""
import numpy as np

from tests import ref64_exposure as R

U = R.U
F = R.F
EPS = F(1e-4)


def level_size(n, k):
    return max(1, n >> (k + 1))


def _input(output, s, ds, p):
    o = np.asarray(output, np.float32).reshape(-1, 4)[:, :3]
    ok = np.isfinite(o) & (o > 0)
    c = np.where(ok, o, np.float32(0)).astype(np.float64)
    x = c * s
    dx = c * ds + U * x
    t = F(p["threshold"])
    if t > 0:
        k = float(np.float32(np.float32(t) * np.float32(p["softness"])))
        den = float(np.float32(np.float32(4.0 * k) + np.float32(1e-4)))
        b = x.max(axis=1)
        db = dx.max(axis=1)
        q0 = np.clip((b - t) + k, 0.0, 2.0 * k)
        dq0 = db + 2 * U * (np.abs(b - t) + np.abs(b - t + k))
        q = q0 * q0 / den
        dq = 2.0 * q0 * dq0 / den + 2 * U * q
        num = np.maximum(q, b - t)
        dnum = np.maximum(dq, db + U * np.abs(b - t))
        dd = np.maximum(b, EPS)
        ddd = np.where(b > EPS, db, 0.0)
        w = num / dd
        dw = dnum / dd + np.abs(w) * ddd / dd + U * np.abs(w)
        y = x * w[:, None]
        dx = dx * np.abs(w)[:, None] + x * dw[:, None] + U * y
        x = y
    return x, dx


def _gather(v, xs, ys):
    h, w = v.shape[:2]
    return v[np.clip(ys, 0, h - 1)[:, None], np.clip(xs, 0, w - 1)[None, :]]


def _down(v, dv, ow, oh, karis):
    i, j = np.arange(ow), np.arange(oh)

    def tap(cx, cy):
        a = [(_gather(v, x, y), _gather(dv, x, y)) for x, y in ((cx - 1, cy - 1), (cx, cy - 1), (cx - 1, cy), (cx, cy))]
        t = sum(q[0] for q in a) / 4.0
        dt = sum(q[1] for q in a) / 4.0 + 2 * U * t
        if not karis:
            return t, dt, None, None
        L, dLr = R.luminance(t)
        dL = dLr + sum(R.W_BT709[k] * dt[..., k] for k in range(3))
        w = 1.0 / (1.0 + L)
        dw = w * w * (dL + U * (1.0 + L)) + U * w
        return t, dt, w, dw

    def group(taps):
        if not karis:
            g = sum(q[0] for q in taps) / 4.0
            return g, sum(q[1] for q in taps) / 4.0 + 2 * U * g
        sw = sum(q[2] for q in taps)[..., None]
        g = sum(q[0] * q[2][..., None] for q in taps) / sw
        dg = sum(q[1] * q[2][..., None] for q in taps) / sw
        dg = dg + sum((q[0] + g) * q[3][..., None] for q in taps) / sw
        return g, dg + 6 * U * g

    o = {(m, n): tap(2 * i - 1 + 2 * m, 2 * j - 1 + 2 * n) for m in range(3) for n in range(3)}
    e = {(m, n): tap(2 * i + 2 * m, 2 * j + 2 * n) for m in range(2) for n in range(2)}
    C = group([e[0, 0], e[1, 0], e[0, 1], e[1, 1]])
    G = [group([o[a, b], o[a + 1, b], o[a, b + 1], o[a + 1, b + 1]]) for a, b in ((0, 0), (1, 0), (0, 1), (1, 1))]
    r = 0.5 * C[0] + 0.125 * sum(g[0] for g in G)
    dr = 0.5 * C[1] + 0.125 * sum(g[1] for g in G) + 3 * U * r
    return r, dr


def _tent(u, du, fw, fh):
    ch, cw = u.shape[:2]
    cx, cy = np.minimum(np.arange(fw) >> 1, cw - 1), np.minimum(np.arange(fh) >> 1, ch - 1)
    t = np.zeros((fh, fw, 3))
    dt = np.zeros((fh, fw, 3))
    for dy, wy in ((-1, 1.0), (0, 2.0), (1, 1.0)):
        for dx, wx in ((-1, 1.0), (0, 2.0), (1, 1.0)):
            t += wy * wx * _gather(u, cx + dx, cy + dy)
            dt += wy * wx * _gather(du, cx + dx, cy + dy)
    t, dt = t / 16.0, dt / 16.0
    return t, dt + 4 * U * t


def pyramid(output, w, h, s, ds, p):
    """float64 (down, up) levels, each a list of (value, bound) arrays (h_k, w_k, 3)."""
    L = int(p["levels"])
    x, dx = _input(output, s, ds, p)
    v, dv = x.reshape(h, w, 3), dx.reshape(h, w, 3)
    down = []
    for k in range(L):
        v, dv = _down(v, dv, level_size(w, k), level_size(h, k), k == 0)
        down.append((v, dv))
    a = F(p["scatter"])
    oma = float(np.float32(1.0) - np.float32(a))
    up = [None] * L
    up[L - 1] = down[L - 1]
    for k in range(L - 2, -1, -1):
        d, dd = down[k]
        t, dt = _tent(*up[k + 1], d.shape[1], d.shape[0])
        r = oma * d + a * t
        up[k] = (r, oma * dd + a * dt + 2 * U * r)
    return [(a_, 2.0 * b_) for a_, b_ in down], [(a_, 2.0 * b_) for a_, b_ in up]


def check_words(words, down, up, mistakes=False):
    """The number of pyramid floats outside the float64 bound (and header / size mismatches as one each)."""
    wd = np.asarray(words, np.float32).reshape(-1)
    u = wd.view(np.uint32)
    L = len(down)
    bad = 0
    sizes = [(v.shape[1], v.shape[0]) for v, _ in down]
    if int(u[0]) != L or any((int(u[1 + 2 * k]), int(u[2 + 2 * k])) != sizes[k] for k in range(L)):
        return 1
    off = 20
    want = sum(4 * sw * sh for sw, sh in sizes) * 2 - 4 * sizes[-1][0] * sizes[-1][1]
    if wd.size != off + want:
        return 1
    for lv in (down, up[:L - 1]):
        for v, dv in lv:
            n = v.shape[0] * v.shape[1]
            got = wd[off:off + 4 * n].reshape(v.shape[0], v.shape[1], 4)
            off += 4 * n
            g = got[..., :3].astype(np.float64)
            bad += int((~np.isfinite(g) | (np.abs(g - v) > dv)).sum()) + int((got[..., 3] != 0).sum())
    return bad


def _bytes(t, dt):
    from tests.ref64_svgf import srgb_encode
    dt = np.where(np.isfinite(dt), dt, np.inf)
    res = []
    for v in (t - dt, t + dt):
        v32 = np.clip(np.nan_to_num(v, nan=0.0, posinf=2.0, neginf=-1.0), -1.0, 2.0).astype(np.float32)
        _, tt, wt = srgb_encode(v32)
        res.append((255.0 * R._srgb(np.clip(v, 0.0, 1.0)) + 0.5, wt))
    (e_lo, w_lo), (e_hi, w_hi) = res
    lo = np.clip(np.floor(e_lo - w_lo - 255.0 * 16 * U), 0, 255).astype(np.int64)
    hi = np.clip(np.floor(e_hi + w_hi + 255.0 * 16 * U), 0, 255).astype(np.int64)
    return lo, hi


def display(output, w, h, op, tm, ev, compensation, p):
    """Per channel (lo, hi) of the bloomed Rgba8 store (n x 3), and the float64 pyramid."""
    o = np.asarray(output, np.float32).reshape(-1, 4)[:, :3]
    if tm:
        y = float(np.float32(np.float32(compensation) - np.float32(ev)))
        s, ds = 2.0 ** y, 2.0 ** y * R.POW2_REL(y)
    else:
        s, ds = 1.0, 0.0
    down, up = pyramid(output, w, h, s, ds, p)
    B, dB = _tent(*up[0], w, h)
    B, dB = B.reshape(-1, 3), dB.reshape(-1, 3)
    if op == 0:
        with np.errstate(invalid="ignore"):
            x = np.nan_to_num(o.astype(np.float64), nan=0.0, posinf=np.inf, neginf=-np.inf)
        dx = np.zeros_like(x)
    else:
        c = np.where(o > 0, o, np.float32(0)).astype(np.float64)
        x, dx = c * s, c * ds + U * c * s
    I = F(p["intensity"])
    if int(p["mode"]) == 0:
        k = float(np.float32(1.0) - np.float32(I))
        xp = k * x + I * B
        dxp = k * dx + I * dB + U * (np.abs(k * x) + np.abs(I * B)) + U * np.abs(xp)
    else:
        xp = x + I * B
        dxp = dx + I * dB + U * np.abs(I * B) + U * np.abs(xp)
    dxp = 2.0 * dxp
    if op == 0:
        t, dt = xp, dxp
    else:
        t, dt = R.transform(xp, dxp, op)
    lo, hi = _bytes(t, dt)
    if op == 0:   # today's store of a NaN channel: sat(NaN) is 0 in both
        nan = np.isnan(o)
        lo, hi = np.where(nan, 0, lo), np.where(nan, 255, hi)
    return lo, hi, down, up
