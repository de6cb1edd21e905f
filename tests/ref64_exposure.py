"""Float64 restatement of exposure and tonemapping (ST_OPT_TONEMAPPING, ST_OPT_AUTO_EXPOSURE; DESIGN.md §2 "Exposure and tonemapping"),
with derived bounds on the f32 evaluation.

- Histogram: L in float64 from the f32 channels, with the rounding of its three products and two sums (gamma(3) sum |c_i x_i|); the bin
  coordinate y = 8 (log2 L + 16), with L's error through d log2 = dL / (L ln 2), log2_x's own bound LOG2_ABS (1 + |log2 L|) (measured in
  test_primitive_bounds) and the rounding of the add and the multiply.  A pixel's bin is decided where y +- bound stays in one bin.
- Metering and adaptation: the rule's doubles are exact here (bin counts and 1/16-multiples below 2^53), so the float64 restatement over
  the same counts gives the same EV bits; adaptation is restated in float32.
- Display: first-order forward error bounds of each operator on exposed x = max(c, 0) 2^(comp - ev) (pow_det(2, y): POW2_REL(y)), doubled
  for the second-order terms; pow_det(u, 2.2) within POW22_REL(u); then the store is monotone, so a byte is decided where the sRGB
  encodings of T +- bound (each with ref64_svgf.srgb_encode's own window) round to the same byte.
"""
import math

import numpy as np

U = 2.0 ** -24
ULP = 2.0 ** -23
LOG2_MID_GREY = math.log2(0.18)
LOG2_ABS = 2.0 ** -21          # log2_x(x) - log2(x) <= LOG2_ABS (1 + |log2 x|)            (test_primitive_bounds)
F = lambda v: float(np.float32(v))
W_BT709 = (F(0.2126), F(0.7152), F(0.0722))
W_BT601 = (0.299, 0.587, 0.114)
A_ACES = np.array([[0.59719, 0.35458, 0.04823], [0.07600, 0.90834, 0.01566], [0.02840, 0.13383, 0.83777]], np.float32).astype(np.float64)
B_ACES = np.array([[1.60475, -0.53108, -0.07367], [-0.10208, 1.10813, -0.00605], [-0.00327, -0.07276, 1.07602]], np.float32).astype(np.float64)
M_AGX = np.array([[0.842479062253094, 0.0784335999999992, 0.0792237451477643], [0.0423282422610123, 0.878468636469772, 0.0791661274605434],
                  [0.0423756549057051, 0.0784336, 0.879142973793104]], np.float32).astype(np.float64)
MI_AGX = np.array([[1.19687900512017, -0.0980208811401368, -0.0990297440797205], [-0.0528968517574562, 1.15190312990417, -0.0989611768448433],
                   [-0.0529716355144438, -0.0980434501171241, 1.15107367264116]], np.float32).astype(np.float64)
AGX_MIN, AGX_MAX, AGX_RANGE = F(-12.47393), F(4.026069), F(16.499999)
AGX_POLY = [F(c) for c in (15.5, -40.14, 31.96, -6.868, 0.4298, 0.1191, -0.00232)]   # n^6 .. n^0
ACES_C = [F(c) for c in (0.0245786, 0.000090537, 0.983729, 0.4329510, 0.238081)]


def gamma(n):
    return n * U / (1 - n * U)


def POW2_REL(y):
    """pow_det(2, y) = exp_det(y log_det(2)): relative bound (test_primitive_bounds)."""
    return (2.0 + 2.0 * np.abs(y) * math.log(2.0)) * ULP


def POW22_REL(u):
    """pow_det(u, 2.2), u in (0, 2]: relative bound (test_primitive_bounds)."""
    return (4.0 + 2.2 * np.abs(np.log(np.where(u > 0, u, 1.0)))) * ULP


# ---- histogram ------------------------------------------------------------------------------------------------------------------

def luminance(rgb, weights=W_BT709):
    x = np.asarray(rgb, np.float64)
    terms = [weights[k] * x[..., k] for k in range(3)]
    L = (terms[0] + terms[1]) + terms[2]
    return L, gamma(3) * (np.abs(terms[0]) + np.abs(terms[1]) + np.abs(terms[2]))


def bins(output, weights=W_BT709):
    """Per pixel (lo, hi): the bins the f32 evaluation can land in (lo == hi: decided); -1 where the pixel does not count."""
    o = np.asarray(output, np.float32).reshape(-1, 4)
    L32 = np.asarray(luminance(o[:, :3])[0], np.float64)
    L, dL = luminance(o[:, :3], weights)
    counts = np.isfinite(L32) & (L32 > 0) & np.isfinite(L) & (L > 0)
    with np.errstate(divide="ignore", invalid="ignore"):
        lg = np.where(counts, np.log2(np.where(counts, L, 1.0)), 0.0)
        dlg = dL / (np.where(counts, L, 1.0) * math.log(2.0)) + LOG2_ABS * (1.0 + np.abs(lg))
    y = (lg + 16.0) * 8.0
    dy = 8.0 * (dlg + U * np.abs(lg + 16.0)) + U * np.abs(y) + 1e-300
    b = lambda v: np.clip(np.floor(v), 0, 255).astype(np.int64)
    lo, hi = np.where(counts, b(y - dy), -1), np.where(counts, b(y + dy), -1)
    return lo, hi


def check_histogram(counts, lo, hi):
    """The device's counts are consistent with the per-pixel ranges: each bin holds at least the pixels decided into it and at most the
    pixels that can land in it.  Returns the number of bins outside."""
    c = np.asarray(counts, np.int64)
    sure = np.bincount(lo[(lo >= 0) & (lo == hi)], minlength=256)
    can = np.zeros(256, np.int64)
    for a, z in zip(lo[lo >= 0], hi[lo >= 0]):
        can[a:z + 1] += 1
    return int(((c < sure) | (c > can)).sum())


# ---- metering and adaptation ------------------------------------------------------------------------------------------------------

def meter(counts, p, state, lower_edge=False, no_window=False, swap=False):
    """(ev, target) float32 of one frame from the bin counts, st_exposure p (8 floats) and the state {ev bits, frames}."""
    c = np.asarray(counts, np.float64)
    n = c.sum()
    lo, hi = (0.0, n) if no_window else (math.floor(float(np.float32(p[4])) * n), math.ceil(float(np.float32(p[5])) * n))
    start = np.concatenate([[0.0], np.cumsum(c)[:-1]])
    k = np.clip(np.minimum(start + c, hi) - np.maximum(start, lo), 0.0, None)
    centre = -16.0 + (np.arange(256) + (0.0 if lower_edge else 0.5)) / 8.0
    ev_prev, first = np.float32(state[0]), state[1] == 0
    f = lambda v: np.float32(v)
    if k.sum() > 0:
        target = f(min(max(float((k * centre).sum() / k.sum() - LOG2_MID_GREY), float(f(p[2]))), float(f(p[3]))))
    else:
        target = f(min(max(0.0, float(f(p[2]))), float(f(p[3])))) if first else ev_prev
    if first:
        return target, target
    up, down = (f(p[7]), f(p[6])) if swap else (f(p[6]), f(p[7]))
    d = f(target - ev_prev)
    if d > up:
        return f(ev_prev + up), target
    if d < -down:
        return f(ev_prev - down), target
    return target, target


# ---- display ----------------------------------------------------------------------------------------------------------------------

def _mat(m, x, dx):
    v = np.einsum("ij,...j->...i", m, x)
    return v, gamma(3) * np.einsum("ij,...j->...i", np.abs(m), np.abs(x)) + np.einsum("ij,...j->...i", np.abs(m), dx)


def transform(x, dx, op, weights=W_BT709, aces_t=False, agx_t=False, agx_pow=True):
    """T(x) in float64 and its first-order bound (doubled), x: (..., 3) exposed channels with bound dx."""
    if op == 1:
        return x, dx
    if op == 2:
        L, dLr = luminance(x, weights)
        dL = dLr + sum(weights[k] * dx[..., k] for k in range(3))
        d = 1.0 + L
        dd = dL + U * d
        t = x / d[..., None]
        return t, 2.0 * ((dx + np.abs(x) * (dd / d)[..., None]) / d[..., None] + U * np.abs(t))
    if op == 3:
        a, b, c, e, g = ACES_C
        A, B = (A_ACES.T, B_ACES.T) if aces_t else (A_ACES, B_ACES)
        v, dv = _mat(A, x, dx)
        N, D = v * (v + a) - b, v * (c * v + e) + g
        w = N / D
        dw_dv = ((2 * v + a) * D - N * (2 * c * v + e)) / D ** 2
        dN, dD = 3 * U * (np.abs(v) * (np.abs(v) + a) + b), 4 * U * (np.abs(v) * (c * np.abs(v) + e) + g)
        dw = np.abs(dw_dv) * dv + (dN + np.abs(w) * dD) / D + U * np.abs(w)
        t, dt = _mat(B, w, dw)
        return t, 2.0 * dt
    if op == 4:
        M, MI = (M_AGX.T, MI_AGX.T) if agx_t else (M_AGX, MI_AGX)
        v, dv = _mat(M, x, dx)
        pos = v > 0
        with np.errstate(divide="ignore", invalid="ignore"):
            l = np.where(pos, np.log2(np.where(pos, v, 1.0)), AGX_MIN)
            dl = np.where(pos, dv / (np.where(pos, v, 1.0) * math.log(2.0)) + LOG2_ABS * (1.0 + np.abs(l)), 0.0)
        dl = np.where(~pos & (dv > 0), np.inf, dl)   # a value at 0 whose sign is not decided: no bound on l
        lc = np.clip(l, AGX_MIN, AGX_MAX)
        n = (lc - AGX_MIN) / AGX_RANGE
        dn = (np.minimum(dl, AGX_MAX - AGX_MIN) + U * np.abs(lc - AGX_MIN)) / AGX_RANGE + U * np.abs(n)
        c6, c5, c4, c3, c2, c1, c0 = AGX_POLY
        p = c6 * n ** 6 + c5 * n ** 5 + c4 * n ** 4 + c3 * n ** 3 + c2 * n ** 2 + c1 * n + c0
        dp_dn = 6 * c6 * n ** 5 + 5 * c5 * n ** 4 + 4 * c4 * n ** 3 + 3 * c3 * n ** 2 + 2 * c2 * n + c1
        terms = np.abs(c6) * n ** 6 + np.abs(c5) * n ** 5 + np.abs(c4) * n ** 4 + np.abs(c3) * n ** 3 + np.abs(c2) * n ** 2 + np.abs(c1) * n + np.abs(c0)
        dp = np.abs(dp_dn) * dn + 12 * U * terms
        u, du = _mat(MI, p, dp)
        uc = np.maximum(u, 0.0)
        if not agx_pow:
            return uc, 2.0 * du
        t = uc ** 2.2
        dt = 2.2 * np.maximum(np.abs(u) + du, 0.0) ** 1.2 * du + t * POW22_REL(uc)
        return t, 2.0 * dt
    raise ValueError(op)


def _srgb(e):
    e = np.clip(e, 0.0, 1.0)
    return np.where(e <= 0.0031308, 12.92 * e, 1.055 * e ** (1.0 / 2.4) - 0.055)


def display(output, op, ev, compensation, after_t=False, **mistakes):
    """Per channel (lo, hi): the bytes the f32 store can produce (lo == hi: decided)."""
    from tests.ref64_svgf import srgb_encode
    o = np.asarray(output, np.float32).reshape(-1, 4)[:, :3]
    c = np.where(o > 0, o, np.float32(0)).astype(np.float64)
    y = float(np.float32(np.float32(compensation) - np.float32(ev)))
    s = 2.0 ** y
    ds = s * POW2_REL(y)
    if after_t:
        t, dt = transform(c, np.zeros_like(c), op, **mistakes)
        t, dt = t * s, dt * s + np.abs(t) * ds + U * np.abs(t) * s
    else:
        x = c * s
        t, dt = transform(x, c * ds + U * x, op, **mistakes)
    dt = np.where(np.isfinite(dt), dt, np.inf)
    lo_v, hi_v = t - dt, t + dt
    # the store is monotone in its input: the extreme bytes come from the ends of the interval, each with the encoding's own window
    res = []
    for v in (lo_v, hi_v):
        v32 = np.clip(np.nan_to_num(v, nan=0.0, posinf=2.0, neginf=-1.0), -1.0, 2.0).astype(np.float32)
        _, tt, wt = srgb_encode(v32)
        e = 255.0 * _srgb(np.clip(v, 0.0, 1.0)) + 0.5
        res.append((e, tt, wt))
    (e_lo, _, w_lo), (e_hi, _, w_hi) = res
    lo = np.clip(np.floor(e_lo - w_lo - 255.0 * 16 * U), 0, 255).astype(np.int64)
    hi = np.clip(np.floor(e_hi + w_hi + 255.0 * 16 * U), 0, 255).astype(np.int64)
    return lo, hi
