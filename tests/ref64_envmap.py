"""The environment map's lookup (st_set_environment_map, DESIGN.md §2 "Environment map") restated in float64 from its definition, with
an error bound derived term by term from the float32 evaluation, and the checks of the three passes that evaluate it (K10's sky
pixels, K13's bounce, K2's miss) on the oracle extension's probe records (oracle_envmap/envmap.cpp documents their layout).

For a float32 direction d (exact input): theta = acos(clamp(d.y)), phi = atan2(d.x, -d.z), u = (phi + rotation) / 2 pi + 0.5,
v = theta / pi, s = u W - 0.5, t = v H - 0.5; the value is the bilinear blend of columns floor(s), floor(s) + 1 (wrapped) and rows
floor(t), floor(t) + 1 (clamped), times the intensity.  The blend is a continuous function of (s, t) (wrapping and clamping keep it so,
the atan2 cut included: u = 0 and u = 1 give the same columns), Lipschitz with constant Ls (the largest difference of horizontally
neighbouring texels in the cells the interval reaches) along s and Lt along t.  So the float32 value lies within
    I (Ls ds + Lt dt + 6 u M) + u I M
of the float64 one, where ds, dt bound the float32 s, t (below), M is the largest texel magnitude of those cells (the three roundings
of each of the two lerp levels) and u = 2^-24 (the product with the intensity).  ds and dt:
    acos_x, atan2_x: ACOS_ULP, ATAN2_ULP float32 ulps of the result (asserted by test_acos_atan2_within_ulp_bound);
    phi + rotation: + u |a|;  x (1 / 2 pi) as a float32 constant: + 2 u |a| / 2 pi;  + 0.5: + u |u|;  x W: + u |u W|;  - 0.5: + u |s|;
    theta x (1 / pi): + 2 u theta / pi;  x H: + u |v H|;  - 0.5: + u |t|.
A texel choice counts as decided when s and t are farther than ds, dt from an integer; there the float32 columns and rows must be the
float64 ones exactly.  The rest are counted as undecided (their values are still checked against the bound above)."""
import numpy as np

U = 2.0 ** -24
ACOS_ULP, ATAN2_ULP = 2.0, 4.0   # measured: 1.24 and 2.99 over test_acos_atan2_within_ulp_bound's sweep
SAFETY = 1.05


def ulp32(x):
    """The float32 ulp at |x| (the spacing above |x| rounded to float32)."""
    return np.spacing(np.abs(np.asarray(x, np.float64)).astype(np.float32)).astype(np.float64)


def coords(d, W, H, rotation):
    """float64 s, t and their bounds ds, dt for float32 directions d (n x 3)."""
    d = np.asarray(d, np.float64)
    theta = np.arccos(np.clip(d[:, 1], -1.0, 1.0))
    phi = np.arctan2(d[:, 0], -d[:, 2])
    a = phi + float(rotation)
    u = a / (2.0 * np.pi) + 0.5
    v = theta / np.pi
    s, t = u * W - 0.5, v * H - 0.5
    ea = ATAN2_ULP * ulp32(phi) + U * np.abs(a)
    eu = ea / (2.0 * np.pi) + 2.0 * U * np.abs(a) / (2.0 * np.pi) + U * np.abs(u)
    ds = SAFETY * (eu * W + U * np.abs(u * W) + U * np.abs(s))
    ev = ACOS_ULP * ulp32(theta) / np.pi + 2.0 * U * theta / np.pi
    dt = SAFETY * (ev * H + U * np.abs(v * H) + U * np.abs(t))
    return s, t, ds, dt


def lookup(tex, intensity, rotation, d):
    """float64 values (n x 3), bounds (n x 3), the float64 texel choice (x0, x1, y0, y1) and a decided mask, for directions d."""
    H, W = tex.shape[:2]
    rgb = np.asarray(tex[..., :3], np.float64)
    s, t, ds, dt = coords(d, W, H, rotation)
    fs, ft = np.floor(s), np.floor(t)
    tx, ty = (s - fs)[:, None], (t - ft)[:, None]
    x0 = np.mod(fs.astype(np.int64), W); x1 = np.mod(x0 + 1, W)
    y0 = np.clip(ft.astype(np.int64), 0, H - 1); y1 = np.clip(ft.astype(np.int64) + 1, 0, H - 1)
    a, b, c, e = rgb[y0, x0], rgb[y0, x1], rgb[y1, x0], rgb[y1, x1]
    top, bot = a + (b - a) * tx, c + (e - c) * tx
    val = (top + (bot - top) * ty) * float(intensity)
    # the cells the intervals [s - ds, s + ds] x [t - dt, t + dt] reach: 3 columns and 3 rows from floor(s - ds), floor(t - dt)
    c0 = np.floor(s - ds).astype(np.int64)
    r0 = np.floor(t - dt).astype(np.int64)
    cols = np.mod(c0[:, None] + np.arange(3)[None, :], W)
    rows = np.clip(r0[:, None] + np.arange(3)[None, :], 0, H - 1)
    blk = rgb[rows[:, :, None], cols[:, None, :]]   # n x 3 rows x 3 cols x 3
    Ls = np.abs(np.diff(blk, axis=2)).max(axis=(1, 2))
    Lt = np.abs(np.diff(blk, axis=1)).max(axis=(1, 2))
    M = np.abs(blk).max(axis=(1, 2))
    I = float(intensity)
    bound = I * (Ls * ds[:, None] + Lt * dt[:, None] + 6.0 * U * M) + U * I * M + 1e-38
    decided = (np.abs(s - np.round(s)) > ds) & (np.abs(t - np.round(t)) > dt)
    return val, bound, np.stack([x0, x1, y0, y1], axis=1), decided


def ratio(got, want, bound):
    """max |got - want| / bound (0 where equal); inf where the bound is exceeded by a non-finite value."""
    err = np.abs(np.asarray(got, np.float64) - want)
    with np.errstate(invalid="ignore", divide="ignore"):
        r = np.where(err == 0, 0.0, err / bound)
    return np.where(np.isfinite(r), r, np.inf)


def check_records(recs, tex, intensity, rotation, inv_pi_f32=float(np.float32(1.0) / np.float32(np.pi))):
    """Checks every probe record (n x 32) against the float64 restatement; returns a dict of the worst bound usage per site, the
    record counts and the undecided count, and a list of failures (empty: all inside)."""
    recs = np.asarray(recs, np.float32)
    site = recs[:, 0].astype(int)
    d = recs[:, 2:5]
    out = {"records": len(recs), "undecided": 0, "worst": 0.0, "sites": {}}
    bad = []
    valid = np.isfinite(recs[:, 5]) & np.isfinite(recs[:, 6])
    k13_light = (site == 2) & (recs[:, 11] == 0.0)
    look = valid & ~k13_light
    val, bnd, choice, decided = lookup(tex, intensity, rotation, d[look]) if look.any() else (np.zeros((0, 3)),) * 2 + (None, None)
    env_f = recs[look, 7:10].astype(np.float64)
    r_env = ratio(env_f, val, bnd)
    if (r_env > 1.0).any():
        bad.append(f"map value outside the bound in {int((r_env.max(axis=1) > 1.0).sum())} of {look.sum()} records (worst {r_env.max():.3g})")
    if look.any():
        got_choice = recs[look, 28:32].astype(np.int64)
        wrong = decided & (got_choice != choice).any(axis=1)
        if wrong.any():
            bad.append(f"{int(wrong.sum())} decided texel choices differ from float64")
        out["undecided"] = int((~decided).sum())
        out["worst"] = float(r_env.max()) if r_env.size else 0.0
    sl = np.flatnonzero(look)
    # K10: diffuse = value / pi within the bound, specular exactly +0
    k = site[sl] == 0
    if k.any():
        rr = recs[sl[k]]
        want = val[k] / np.pi
        b = bnd[k] / np.pi + np.abs(val[k]) * abs(inv_pi_f32 - 1.0 / np.pi) + U * np.abs(want) * 2.0
        r = ratio(rr[:, 22:25], want, b)
        out["sites"]["k10"] = float(r.max())
        if (r > 1.0).any(): bad.append(f"K10 diffuse outside the bound (worst {r.max():.3g})")
        if (rr[:, 25:28].view(np.uint32) != 0).any(): bad.append("K10 specular sky sample is not +0")
    # K13 miss: the radiance is the map's value itself
    k = site[sl] == 1
    if k.any():
        rr = recs[sl[k]]
        if (rr[:, 22:25].view(np.uint32) != rr[:, 7:10].view(np.uint32)).any(): bad.append("K13 miss radiance is not the map value")
        out["sites"]["k13_miss"] = float(r_env[k].max())
    # K13 hit: the sky-or-light decision, and the sky draw's radiance
    hit = site == 2
    if hit.any():
        rr = recs[hit]
        draw, sky = rr[:, 10], rr[:, 11] == 1.0
        want_sky = (draw < 0) | (draw < np.float32(0.25))
        if (want_sky != sky).any(): bad.append(f"K13 sky-or-light decision differs in {int((want_sky != sky).sum())} of {len(rr)} records")
    k = site[sl] == 2
    if k.any():
        rr = recs[sl[k]]
        n, dd = rr[:, 12:15].astype(np.float64), rr[:, 2:5].astype(np.float64)
        vis, base, em = rr[:, 15:16].astype(np.float64), rr[:, 16:19].astype(np.float64), rr[:, 19:22].astype(np.float64)
        dot = (n * dd).sum(axis=1, keepdims=True)
        f = 4.0 * vis * base / np.pi
        want = val[k] * dot * f + em
        b = bnd[k] * np.abs(dot) * f + np.abs(val[k]) * (3.0 * U * np.linalg.norm(n, axis=1, keepdims=True) * np.linalg.norm(dd, axis=1, keepdims=True)) * f \
            + 8.0 * U * np.abs(val[k] * dot * f) + U * np.abs(want) + 1e-38
        r = ratio(rr[:, 22:25], want, b)
        out["sites"]["k13_sky"] = float(r.max())
        if (r > 1.0).any(): bad.append(f"K13 sky-draw radiance outside the bound (worst {r.max():.3g})")
    # K2: colour after = colour before + throughput x value
    k = site[sl] == 3
    if k.any():
        rr = recs[sl[k]]
        thr, before = rr[:, 12:15].astype(np.float64), rr[:, 16:19].astype(np.float64)
        want = before + thr * val[k]
        b = np.abs(thr) * bnd[k] + U * np.abs(thr * val[k]) + U * np.abs(want) + 1e-38
        r = ratio(rr[:, 22:25], want, b)
        out["sites"]["k2"] = float(r.max())
        if (r > 1.0).any(): bad.append(f"K2 colour outside the bound (worst {r.max():.3g})")
    return out, bad
