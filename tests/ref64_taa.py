"""Float64 restatement of ST_OPT_TEMPORAL_AA (DESIGN.md §2 "Temporal anti-aliasing"), stage by stage, with a derived per-pixel bound.

`check_camera` restates the jittered camera: the projection jittered by J(f) as the rule says, times the inverse transform, against the
serialised record, and the point the record's ray through pixel p reaches, projected through the unjittered float64 camera, against
p + 0.5 + J(f).

`check_resolve` restates the resolve from its inputs (the composed colours, the velocity map, the G-buffer depth, last frame's history,
the jittered cameras) with the oracle's per-pixel record (oracle_taa orc_taa_resolve's probe) supplying the float32 value of each stage's
input, so that every stage is bounded on its own: the history position q, the tonemapped colour t, the Catmull-Rom sample, the clip, the
blend and the inverse tonemap.  u = 2^-24 is the float32 unit roundoff; each bound counts the roundings of the float32 evaluation times
the magnitudes they act on.

Three discrete choices are undecided when the float64 value sits within its bound of the edge, and then accepted either way: whether q is
on screen, floor(q) for the count, and whether the clip engages.  Their counts are returned."""
import numpy as np

U = 2.0 ** -24
TINY = 2.0 ** -140   # absolute slack for float32 subnormals, whose relative spacing exceeds u


def radical_inverse(k, base):
    r, f = 0.0, 1.0 / base
    while k > 0:
        r += f * (k % base)
        k //= base
        f /= base
    return r


def jitter(frame):
    """J(frame) as the rule states it: the radical inverses rounded to float32, minus 0.5 (float64)."""
    k = ((frame - 1) % 16) + 1
    return np.array([float(np.float32(radical_inverse(k, 2))) - 0.5, float(np.float32(radical_inverse(k, 3))) - 0.5])


def _m(a16):
    return np.asarray(a16, np.float64).reshape(4, 4).T   # column-major 16 floats -> row-major matrix


def check_camera(transform16, projection16, w, h, frame, record40):
    """Returns the largest error of the jittered projection_view, relative to its largest entry, and of the screen position (pixels)
    of every pixel's ray; raises past the bounds (64 u relative, 2^-10 pixel)."""
    T, P = _m(transform16), _m(projection16).copy()
    j = jitter(frame)
    P[0, :] += (-2.0 * j[0] / w) * P[3, :]
    P[1, :] += (2.0 * j[1] / h) * P[3, :]
    want = P @ np.linalg.inv(T)
    got = _m(np.asarray(record40, np.float32)[:16])
    rel = float(np.abs(got - want).max() / np.abs(want).max())
    # each pixel's ray (record ndc_to_world at the jittered pixel centre) lands at p + 0.5 + J(f) through the unjittered camera
    n2w = _m(np.asarray(record40, np.float32)[16:32])
    pv = _m(projection16) @ np.linalg.inv(T)
    ys, xs = np.mgrid[0:h, 0:w]
    ndc = np.stack([(xs + 0.5) * 2.0 / w - 1.0, -((ys + 0.5) * 2.0 / h - 1.0), np.full(xs.shape, 0.5), np.ones(xs.shape)], -1)
    world = ndc @ n2w.T
    world = world / world[..., 3:4]
    clip = world @ pv.T
    sx = (clip[..., 0] / clip[..., 3] * 0.5 + 0.5) * w
    sy = (-clip[..., 1] / clip[..., 3] * 0.5 + 0.5) * h
    px = float(max(np.abs(sx - (xs + 0.5 + j[0])).max(), np.abs(sy - (ys + 0.5 + j[1])).max()))
    assert rel <= 64 * U and px <= 2.0 ** -10, f"frame {frame}: jittered camera off by {rel:.3g} (relative) / {px:.3g} px"
    return rel, px


def _tonemap(c):
    return c / (1.0 + c.max(-1, keepdims=True))


def _ycocg(c):
    r, g, b = c[..., 0], c[..., 1], c[..., 2]
    return np.stack([0.25 * r + 0.5 * g + 0.25 * b, 0.5 * r - 0.5 * b, -0.25 * r + 0.5 * g - 0.25 * b], -1)


def _rgb(v):
    y, co, cg = v[..., 0], v[..., 1], v[..., 2]
    return np.stack([y - cg + co, y + cg, y - cg - co], -1)


def _cr(f):
    return np.stack([f * (-0.5 + f * (1.0 - 0.5 * f)), 1.0 + f * f * (-2.5 + 1.5 * f), f * (0.5 + f * (2.0 - 1.5 * f)), f * f * (-0.5 + 0.5 * f)], -1)


def _fail(what, bad, got, want, bound):
    idx = np.flatnonzero(bad)[:4]
    raise AssertionError(f"{what}: {int(bad.sum())} values outside the bound; first at {idx.tolist()}: got {got.reshape(-1)[idx].tolist()} "
                         f"want {want.reshape(-1)[idx].tolist()} bound {bound.reshape(-1)[idx].tolist()}")


def check_resolve(w, h, frame, probe, depth, vel, cam_curr40, cam_prev40, hist_in, hist_out, output):
    """One resolved frame.  probe: (h * w, 24) records; depth: G-buffer d0.x (h * w); vel: velocity map (h * w, 4); cam_*40: the jittered
    camera records; hist_in / hist_out / output: (h * w, 4).  Returns {"worst": largest error / bound, "undecided_*": counts}."""
    pr = np.asarray(probe, np.float64).reshape(h, w, 24)
    hin = np.asarray(hist_in, np.float64).reshape(h, w, 4)
    J, Jp = jitter(frame), jitter(frame - 1)
    ys, xs = np.mgrid[0:h, 0:w].astype(np.float64)
    stats = {"worst": 0.0, "undecided_onscreen": 0, "undecided_floor": 0, "undecided_clip": 0}

    def within(what, got, want, bound):
        got, want, bound = np.asarray(got, np.float64), np.asarray(want, np.float64), np.asarray(bound, np.float64)
        err = np.abs(got - want)
        bound = bound + TINY
        bad = ~(err <= bound)
        if bad.any():
            _fail(what, bad, got, want, bound)
        stats["worst"] = max(stats["worst"], float(np.where(bound > 0, err / np.maximum(bound, 1e-300), 0.0).max()))

    # stage 1: the history position
    q32 = pr[..., 0:2]
    hit = np.asarray(depth).reshape(h, w) != 0.0
    v = np.asarray(vel, np.float64).reshape(h, w, 4)
    q_hit = np.stack([xs + 0.5 - v[..., 0] - (J[0] - Jp[0]), ys + 0.5 - v[..., 1] - (J[1] - Jp[1])], -1)
    n2w, pvp = _m(np.asarray(cam_curr40, np.float32)[16:32]), _m(np.asarray(cam_prev40, np.float32)[:16])
    sx, sy = xs + 0.5 - J[0], ys + 0.5 - J[1]
    nx, ny = sx * 2.0 / w - 1.0, -(sy * 2.0 / h - 1.0)
    def proj(z):
        p = np.stack([nx, ny, np.full(nx.shape, z), np.ones(nx.shape)], -1) @ n2w.T
        return p[..., :3] / p[..., 3:4]
    d = proj(np.float64(np.float32(1.1920929e-7))) - proj(1.0)
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    clip = np.concatenate([d, np.zeros(d.shape[:-1] + (1,))], -1) @ pvp.T
    q_sky = np.stack([(clip[..., 0] / clip[..., 3] * 0.5 + 0.5) * w + Jp[0], (-clip[..., 1] / clip[..., 3] * 0.5 + 0.5) * h + Jp[1]], -1)
    q64 = np.where(hit[..., None], q_hit, q_sky)
    # hits: three roundings on values below |p| + |v| + 1; sky: the camera ray and the projection (about 60 roundings on values of the
    # matrices' size), taken as 2^-12 of the frame size
    mag = np.abs(np.stack([xs, ys], -1)) + np.abs(v[..., 0:2]) + 2.0
    eq = np.where(hit[..., None], 8 * U * mag, 2.0 ** -12 * (w + h))
    sky_ok = hit | (clip[..., 3] > 1e-6)
    within("q", np.where(sky_ok[..., None], q32, 0.0), np.where(sky_ok[..., None], q64, 0.0), eq)
    # discrete choices of stage 1 (on q64 and its bound; the float32 q decides where undecided)
    on64 = (q64[..., 0] >= 0) & (q64[..., 1] >= 0) & (q64[..., 0] < w) & (q64[..., 1] < h)
    edge = np.minimum(np.minimum(np.abs(q64[..., 0]), np.abs(q64[..., 0] - w)), np.minimum(np.abs(q64[..., 1]), np.abs(q64[..., 1] - h)))
    und_on = (edge <= eq.max(-1)) | ~sky_ok
    ok32 = pr[..., 2] != 0
    bad = ~und_on & (on64 != ok32) & hit
    if bad.any():
        _fail("on screen", bad, ok32, on64, eq[..., 0])
    stats["undecided_onscreen"] = int((und_on & (on64 != ok32)).sum())
    fr = q64 - np.floor(q64)
    und_fl = ok32 & ((np.minimum(fr, 1 - fr) <= eq).any(-1)) & (np.floor(q64) != np.floor(q32)).any(-1)
    stats["undecided_floor"] = int(und_fl.sum())
    fx, fy = np.clip(np.floor(q32[..., 0]), 0, w - 1).astype(int), np.clip(np.floor(q32[..., 1]), 0, h - 1).astype(int)
    n_want = np.where(ok32, hin[fy, fx, 3], 0.0)
    n_want = np.where(n_want > 0, n_want, 0.0)
    n32 = pr[..., 3]
    assert (n32 == n_want).all(), f"frame {frame}: count at floor(q) differs at {int((n32 != n_want).sum())} pixels"
    # stage 2: the tonemapped colour and the box
    c = pr[..., 18:21]
    t64 = _tonemap(c)
    within("t", pr[..., 9:12], t64, 4 * U * np.abs(t64) + 1e-300)
    cp = np.pad(c, ((1, 1), (1, 1), (0, 0)), mode="edge")
    nb = np.stack([_ycocg(_tonemap(cp[dy:dy + h, dx:dx + w])) for dy in range(3) for dx in range(3)], 0)
    lo, hi = nb.min(0), nb.max(0)
    within("box", np.concatenate([pr[..., 12:15], pr[..., 15:18]], -1), np.concatenate([lo, hi], -1), 16 * U * (np.abs(np.concatenate([lo, hi], -1)) + 1.0))
    # stage 3: the Catmull-Rom history sample at the float32 q
    acc = n32 > 0
    u_ = q32 - 0.5
    f0 = np.floor(u_)
    wx, wy = _cr(u_[..., 0] - f0[..., 0]), _cr(u_[..., 1] - f0[..., 1])
    hs = np.zeros((h, w, 3))
    absw = np.zeros((h, w))
    for j in range(4):
        yy = np.clip(f0[..., 1].astype(int) - 1 + j, 0, h - 1)
        for k in range(4):
            xx = np.clip(f0[..., 0].astype(int) - 1 + k, 0, w - 1)
            hs += (wx[..., k] * wy[..., j])[..., None] * hin[yy, xx, :3]
            absw += np.abs(wx[..., k] * wy[..., j]) * np.abs(hin[yy, xx, :3]).max(-1)
    bound_h = 48 * U * (absw + 1.0)
    # stage 4: the clip (its engagement undecided within the sample's bound over the box's half extent)
    cc, e = 0.5 * (hi + lo), 0.5 * (hi - lo) + float(np.float32(1e-8))
    dd = _ycocg(hs) - cc
    m = np.abs(dd / e).max(-1)
    und_cl = acc & (np.abs(m - 1.0) <= 2 * bound_h / e.min(-1) + 1e-6)
    eng32 = pr[..., 4] != 0
    eng64 = m > 1.0
    bad = acc & ~und_cl & (eng32 != eng64)
    if bad.any():
        _fail("clip engagement", bad, eng32, eng64, m)
    stats["undecided_clip"] = int((und_cl & (eng32 != eng64)).sum())
    with np.errstate(invalid="ignore", divide="ignore"):
        clipped = _rgb(cc + dd / np.where(m > 0, m, 1.0)[..., None])
    h64 = np.where(acc[..., None], np.where(eng32[..., None], clipped, hs), t64)
    bound_c = np.where(eng32, 3 * bound_h + 24 * U * (np.abs(cc).max(-1) + e.max(-1) + 1.0), bound_h)
    bound_hh = np.where(acc, bound_c, 4 * U * np.abs(t64).max(-1))
    within("history sample", pr[..., 6:9], h64, bound_hh[..., None])
    # stage 5: the blend, the count and the stored history
    alpha = np.maximum(1.0 / (n32 + 1.0), float(np.float32(0.1)))
    r64 = (1.0 - alpha)[..., None] * pr[..., 6:9] + alpha[..., None] * pr[..., 9:12]
    ho = np.asarray(hist_out, np.float64).reshape(h, w, 4)
    within("resolved", ho[..., :3], r64, 6 * U * (np.abs(r64) + np.abs(pr[..., 6:9]) + np.abs(pr[..., 9:12])) + 1e-300)
    assert (ho[..., 3] == np.minimum(n32 + 1.0, 16.0)).all(), f"frame {frame}: stored counts"
    # stage 6: the inverse tonemap of the stored value
    r32 = ho[..., :3]
    mr = r32.max(-1, keepdims=True)
    out64 = r32 / (1.0 - mr)
    o = np.asarray(output, np.float64).reshape(h, w, 4)
    within("output", o[..., :3], out64, 6 * U * np.abs(out64) * (1.0 + mr / np.maximum(1.0 - mr, 1e-300)) + 1e-300)
    return stats
