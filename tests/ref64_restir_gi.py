"""Float64 restatement of the ReSTIR GI reprojection (K11), GI temporal resampling (K14), GI spatial merge (K17) and GI resolving
(K19), with a per-value error bound for either arithmetic tier.

Written from the reference's definitions (paths relative to the reference tree), not from the CUDA kernels or the oracle:
  * K11 `gi_reprojection::main`           strolle-shaders/src/gi_reprojection.rs:4-51
  * K14 `gi_temporal_resampling::main`    strolle-shaders/src/gi_temporal_resampling.rs:4-156; `Mis::gi_temporal`
                                          strolle-gpu/src/reservoir/mis.rs:67-95
  * K17 `gi_spatial_resampling::sample`   strolle-shaders/src/gi_spatial_resampling.rs:225-314
  * K19 `gi_resolving::main`              strolle-shaders/src/gi_resolving.rs:4-67
  * `GiReservoir::read` / `write`, `GiSample::{exists, pdf, dir, cosine, spec_brdf}`   strolle-gpu/src/reservoir/gi.rs:19-57, :93-133
  * `Reservoir::update` / `merge` / `clamp_m` / `clamp_w` / `norm`   strolle-gpu/src/reservoir.rs:24-79
  * `Frame::is_gi_tracing` = frame % 6 < 4 (strolle-gpu/src/frame.rs); `got_checkerboard_at` strolle-gpu/src/utils.rs:41-43
Everything shared with the DI restatement (the running-error numbers `Num`, `Mis::eval`, `Reservoir::update`'s decision, the camera,
G-buffer and hit, the specular BRDF, the white noise, the half-width grid and the octahedral encoding) is imported from
tests/ref64_restir.py, whose docstring states the arithmetic model and the bounds.

What is new here:
  * A GI reservoir is 16 words: radiance, M | v1, w | v2, pdf | oct(v2n), confidence, rng bits.  Every load decodes the normal and
    every store re-encodes it, so a stored normal is encode(decode(e)) of the encoding it came from, bounded through `Num` and never
    compared bit for bit.  Normal::encode's fold (n.z >= 0) and its copysigns are decisions: where one is within its bound (an
    axis-aligned normal has exact zeros there, which the bound cannot tell from tiny values) every consistent encoding is admitted
    and the stored one must match one of them (counted as "seam").  Normal::decode's copysign on a bounded input moves the result by
    at most twice the fold, which is added to the bound.  An empty reservoir's normal is encode(0) = NaN, expected as NaN.
  * `GiSample::exists` compares the stored v2 (exact) with 0; -0 counts as 0.  The pdf, cosine and specular term are `Num`
    expressions on the bounded hit point and the exact stored fields.  The specular `n.l <= 0 || n.v <= 0` early-out is a decision:
    where it is within its bound a pdf that depends on it leaves its pixel uncompared (counted under "specular"), and K19 accepts
    either 0 or the value, as K10 does.
  * K14's radiance-distance test `|lhs - rhs| > 0.33` on validation frames is decided where its margin exceeds the distance's bound;
    otherwise both confidences (0 and 1) are accepted and the pixel is counted under "distance".
  * K14 on validation frames: Reservoir::merge's M = (0 + (M - 1)) + 1 and norm_avg's denominator pdf * M act on exact f32 inputs,
    so they are evaluated in f32 here (exact); `pdf * M == 0` is then decided.
  * `rng * W < weight` (Reservoir::update) is the DI rule: an undecided update enumerates both outcomes.
  * `round()` of the reprojection acts on exact inputs.  The restatement asserts that no reprojected position lies outside the
    frame: the kernel guards `idx < w h`, the reference does not.
  * K17 merges only where the texel's rhs_idx is nonzero *and* rhs_idx - 1 < w h.  The reference reads any nonzero index; the
    kernel's guard reads nothing past the frame and passes the lhs through.  This is a documented deviation: K15 never writes such
    an index, so it only matters for corrupted texels.
"""
import numpy as np

from tests.ref64_restir import (LUMA, PI, Num, WhiteNoise, _decide, _f32c, _mis_eval, _round_u, dot3, half_grid_pairs, hit, norm3,
                                oct_encode, specular, stack3, where)

# Plausible misreadings of the reference, each of which the oracle chain must catch (tests/test_restir_gi_reference.py).  "k14_m64"
# (M clamped at 64) is not among them: GI M stays far below 64 in every oracle run, so the GPU edge test, which injects M at 127,
# 128, 129 and 1e6, is where it must be caught.
MUTATIONS = ("k11_floor", "k14_distance_squared", "k14_phase_frame", "k14_norm_mis_validation", "k17_no_jacobian",
             "k17_rhs_v1", "no_w_clamp", "k19_no_metallic", "k19_source_1")

M_CLAMP = 128.0      # GiReservoir rhs.clamp_m (gi_temporal_resampling.rs:68)
W_CLAMP = 5.0        # clamp_w (gi_temporal_resampling.rs:154, gi_spatial_resampling.rs:302)
DISTANCE = _f32c(0.33)


def tracing_frame(frame):
    return frame % 6 < 4


def resolving_source(frame, mutation=None):
    """The buffer K19 copies into gi_reservoirs[0]: the spatial merge's output on odd tracing frames, the temporal one otherwise."""
    if mutation != "k19_source_1" and tracing_frame(frame) and frame % 2 == 1:
        return "gi_reservoirs_2"
    return "gi_reservoirs_1"


def gi_fields(res):
    """GiReservoir::read (gi.rs:19-40) of an (N, 16) buffer, as exact f32 words: rad (N, 3), m, v1 (N, 3), w, v2 (N, 3), pdf,
    enc (N, 2) (the encoded v2n), conf, rng (u32)."""
    r = np.asarray(res, np.float32).reshape(-1, 16)
    return dict(rad=r[:, 0:3], m=r[:, 3], v1=r[:, 4:7], w=r[:, 7], v2=r[:, 8:11], pdf=r[:, 11], enc=r[:, 12:14], conf=r[:, 14],
                rng=r[:, 15].view(np.uint32))


def _sub(f, i):
    return {k: v[i] for k, v in f.items()}


def _zero_fields(n):
    """GiReservoir::default: every field zero; its normal (0, 0, 0) stores as NaN."""
    z3 = np.zeros((n, 3), np.float32)
    return dict(rad=z3, m=np.zeros(n, np.float32), v1=z3, w=np.zeros(n, np.float32), v2=z3, pdf=np.zeros(n, np.float32),
                enc=np.full((n, 2), np.nan, np.float32), conf=np.zeros(n, np.float32), rng=np.zeros(n, np.uint32))


def _pick(mask, a, b):
    """Per-pixel choice between two field dicts (the same keys)."""
    return {k: np.where(mask.reshape((-1,) + (1,) * (np.ndim(a[k]) - 1)), a[k], b[k]) for k in a}


# ---- octahedral round trip ---------------------------------------------------------------------------------------------------

def oct_decode_num(e):
    """Normal::decode (normal.rs) of a bounded encoding e (Num (N, 2)): (Num (N, 3), decided).  Where a coordinate is within its
    bound of 0 the sign copysign gives the fold t is not known, but both results lie within 2 t of each other: that is added to the
    coordinate's bound, so the decode is always decided."""
    fast = e.fast
    mx, my = e.col(0) * 2.0 - 1.0, e.col(1) * 2.0 - 1.0
    nz = (1.0 - mx.abs()) - my.abs()
    t = (-nz).maximum(0.0)

    def fold(m):
        x = m - Num(np.copysign(t.v, m.v), t.e, fast)
        return Num(x.v, x.e + np.where(np.abs(m.v) <= m.e, 2.0 * (t.v + t.e), 0.0), fast)
    return norm3(stack3(fold(mx), fold(my), nz)), np.ones(len(mx.v), bool)


def _encode_alts(n, valid):
    """Normal::encode (normal.rs:9-23) of a bounded direction: every encoding consistent with the fold (n.z >= 0) and, below the
    equator, the copysigns of x and y, as a list of (Num (N, 2), mask).  A decision within its bound (an axis-aligned normal has exact
    zeros there) admits both of its branches; NaN stays NaN."""
    fast = n.fast
    s = (n.col(0).abs() + n.col(1).abs()) + n.col(2).abs()
    q = n / s.x3()
    x, y, zc = q.col(0), q.col(1), q.col(2)
    nan = np.isnan(n.v).any(-1)
    zu = np.abs(zc.v) <= zc.e
    up = zc.v >= 0
    st = lambda a, b: Num(np.stack([a.v, b.v], -1), np.stack([a.e, b.e], -1), fast)
    alts = [(st(x * 0.5 + 0.5, y * 0.5 + 0.5), valid & (up | zu | nan))]
    tx, ty = 1.0 - y.abs(), 1.0 - x.abs()
    for sx in (1.0, -1.0):
        for sy in (1.0, -1.0):
            okx = (np.abs(x.v) <= x.e) | (np.sign(x.v) == sx)
            oky = (np.abs(y.v) <= y.e) | (np.sign(y.v) == sy)
            enc = st(Num(sx * tx.v, tx.e, fast) * 0.5 + 0.5, Num(sy * ty.v, ty.e, fast) * 0.5 + 0.5)
            alts.append((enc, valid & ~nan & (~up | zu) & okx & oky))
    return alts


def oct_roundtrip(enc, fast):
    """encode(decode(e)) of an (N, 2) encoding: exact words (array), or the alternatives [(Num (N, 2), mask)] of an earlier round
    trip.  Returns (alternatives, decided): decided is False where Normal::decode's copysign was within its bound (not compared)."""
    if not isinstance(enc, list):
        enc = [(Num(np.asarray(enc, np.float32).astype(np.float64), 0.0, fast), np.ones(len(enc), bool))]
    out, dec = [], np.ones(len(enc[0][1]), bool)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        for e, valid in enc:
            n, dec1 = oct_decode_num(e)
            dec &= dec1 | ~valid | np.isnan(e.v).any(-1)
            out += _encode_alts(n, valid)
    return out, dec


def nan_enc(n, fast):
    """The stored normal of a reservoir whose v2n is (0, 0, 0): NaN."""
    return [(Num(np.full((n, 2), np.nan), 0.0, fast), np.ones(n, bool))]


def pick_enc(mask, a, b):
    return [(e, m & mask) for e, m in a] + [(e, m & ~mask) for e, m in b]


# ---- GiSample --------------------------------------------------------------------------------------------------------------

def exists(v2):
    """GiSample::exists: v2 != (0, 0, 0) on exact words (-0 == 0)."""
    return ~(np.asarray(v2, np.float32) == 0).all(-1)


def gi_dir(v2, point):
    return norm3(Num(np.asarray(v2, np.float64), 0.0, point.fast) - point)


def gi_cosine(v2, ht):
    return dot3(gi_dir(v2, ht["point"]), ht["g"]["normal"]).maximum(0.0)


def _luma(c):
    return (c.col(0) * LUMA[0] + c.col(1) * LUMA[1]) + c.col(2) * LUMA[2]


def gi_pdf(rad, v2, ht):
    """GiSample::pdf (gi.rs:98-112) for per-pixel samples and hits: luma(radiance) cosine (luma(diffuse) + luma(specular)) with the
    base colour set to 1, 0 where the sample does not exist.  Returns (pdf, specular undecided)."""
    fast = ht["point"].fast
    g = dict(ht["g"], base=Num(np.ones(ht["g"]["base"].v.shape), 0.0, fast))
    d = gi_dir(v2, ht["point"])
    cos = dot3(d, g["normal"]).maximum(0.0)
    diff = (1.0 - g["metallic"]) / PI
    diff_l = (diff * LUMA[0] + diff * LUMA[1]) + diff * LUMA[2]
    spec, und = specular(g, d, -ht["dir"])
    pdf = (_luma(Num(np.asarray(rad, np.float64), 0.0, fast)) * cos) * (diff_l + _luma(spec))
    ex = exists(v2)
    return where(ex, pdf, Num(np.zeros(len(ex)), 0.0, fast)), und & ex


# ---- expected reservoirs and their check ---------------------------------------------------------------------------------------

def _cand(allowed, rad, m, v1, w, v2, pdf, enc, conf, rng, fold_und=None):
    """One admissible outcome per pixel: value (N, 16) and bound (N, 16) (0: exact) of every word but the normal, the rng bits, and
    the normal's admissible encodings `enc` (oct_roundtrip's alternatives); the normal is not compared where `fold_und`."""
    n = len(allowed)
    v, e = np.zeros((n, 16)), np.zeros((n, 16))
    for cols, x in ((slice(0, 3), rad), (3, m), (slice(4, 7), v1), (7, w), (slice(8, 11), v2), (11, pdf), (14, conf)):
        if isinstance(x, Num):
            v[:, cols], e[:, cols] = x.v, x.e
        else:
            v[:, cols] = np.asarray(x, np.float64)
    fold_und = np.zeros(n, bool) if fold_und is None else fold_und
    return dict(v=v, e=e, rng=np.asarray(rng, np.uint32), enc=enc, fold_und=fold_und,
                seam=sum(mk.astype(int) for _, mk in enc) > 1, allowed=allowed)


def stored(f, fast, enc=None, **over):
    """The candidate GiReservoir::write makes of fields `f` (exact words) with the normal through the round trip; `over` replaces
    fields by bounded values.  Returns (candidate pieces, fold decided)."""
    enc_out, dec = oct_roundtrip(f["enc"] if enc is None else enc, fast)
    out = dict(rad=f["rad"], m=f["m"], v1=f["v1"], w=f["w"], v2=f["v2"], pdf=f["pdf"], enc=enc_out, conf=f["conf"], rng=f["rng"])
    out.update(over)
    return out, dec


def _ratio_of(gv, v, e):
    with np.errstate(invalid="ignore", divide="ignore"):
        err = np.abs(gv - v)
        rk = np.where(err == 0, 0.0, err / e)
    return np.where(np.isnan(v), np.where(np.isnan(gv), 0.0, np.inf), np.where(np.isnan(rk), np.inf, rk))


def check_gi(got, r, what):
    """Every pixel of r["idx"] (but the skipped ones) matches one admissible candidate: NaN where NaN is expected, the rng bits
    exactly, the normal one of its admissible encodings, every other word within its bound (bit for bit where the bound is 0).
    Returns the largest error / bound ratio."""
    g = np.asarray(got, np.float32).reshape(-1, 16)[r["idx"]]
    gv = g.astype(np.float64)
    grng = g[:, 15].view(np.uint32)
    ok = r["skip"].copy()
    best = np.full(len(g), np.inf)
    for c in r["cands"]:
        rk = _ratio_of(gv, c["v"], c["e"])
        rk[:, 15] = np.where(grng == c["rng"], 0.0, np.inf)
        re = np.full(len(g), np.inf)
        for ev, mk in c["enc"]:
            re = np.where(mk, np.minimum(re, _ratio_of(gv[:, 12:14], ev.v, ev.e).max(1)), re)
        rk[:, 12] = np.where(c["fold_und"], 0.0, re)
        rk[:, 13] = 0.0
        ratio = rk.max(1)
        good = c["allowed"] & (ratio <= 1.0) & ~r["skip"]
        best = np.where(good, np.minimum(best, ratio), best)
        ok |= good
    if not ok.all():
        i = np.flatnonzero(~ok)[:3]
        raise AssertionError(f"{what}: {int((~ok).sum())}/{len(ok)} pixels match no admissible outcome; first pixels "
                             f"{r['idx'][i].tolist()}: got {g[i].tolist()}")
    best = best[~r["skip"]]
    return float(best.max()) if len(best) else 0.0


def check_untouched(got, before, keep, what):
    """The pixels `keep` (flat indices) of a (N, 16) reservoir buffer are as they were, bit for bit."""
    a = np.asarray(got, np.float32).reshape(-1, 16)[keep].view(np.uint32)
    b = np.asarray(before, np.float32).reshape(-1, 16)[keep].view(np.uint32)
    assert (a == b).all(), f"{what}: {int((a != b).any(1).sum())} pixels it must leave were written"


def tight(r, cols):
    """[tightly bounded (below 1e-3 relative), finite nonzero] over the columns `cols` of the outcome of each decided pixel."""
    t = n = 0
    sel0 = ~r["skip"] & ~r["any_undecided"]
    for c in r["cands"]:
        sel = c["allowed"] & sel0
        v, e = c["v"][sel][:, cols], c["e"][sel][:, cols]
        fin = np.isfinite(v) & (v != 0)
        n += int(fin.sum()); t += int((e[fin] < 1e-3 * np.abs(v[fin])).sum())
    return [t, n]


def _result(idx, cands, und, skip=None, **extra):
    any_und = np.zeros(len(idx), bool)
    for v in und.values():
        any_und |= v
    skip = np.zeros(len(idx), bool) if skip is None else skip
    # pixels whose stored normal may take more than one encoding (a fold sign of an exact zero): compared with each of them
    seam = np.zeros(len(idx), bool)
    for c in cands:
        seam |= c["allowed"] & c["seam"]
    return dict(idx=idx, cands=cands, undecided={k: int(v.sum()) for k, v in und.items()}, any_undecided=any_und, skip=skip,
                seam=int(seam.sum()), **extra)


# ---- K11: reprojection -------------------------------------------------------------------------------------------------------

def _reproject(reproj, idx, w, h, mutation=None):
    """(has a previous position, its flat index) of the pixels idx: Reprojection::prev_pos_round, reprojection.rs:46-48."""
    rp = np.asarray(reproj, np.float32).reshape(-1, 4)[idx]
    has = rp[:, 2] > 0
    if mutation == "k11_floor":
        rx, ry = (np.clip(np.nan_to_num(np.floor(rp[:, k].astype(np.float64))), 0, 2.0 ** 32 - 1).astype(np.int64) for k in (0, 1))
    else:
        rx, ry = _round_u(rp[:, 0]), _round_u(rp[:, 1])
    assert ((rx < w) & (ry < h))[has].all(), "reprojected position outside the frame"
    return has, np.where(has, ry * w + rx, 0), rx, ry


def gi_reprojection(n2w, w, h, d0, d1, reproj, res0, fast, mutation=None, xs=None, ys=None):
    """K11 for the pixels with a surface (of all pixels, or of (xs, ys)): gi_reservoirs[0] at round() of the reprojection (or the
    default reservoir where there is none), confidence 1, v1 = the hit point.  Returns the restatement plus `fields` (the reservoir
    K14's inline form hands on, with its normal still encoded as it was read), `point`, `has` and `sky` (flat indices left alone)."""
    if xs is None:
        ys, xs = (a.reshape(-1) for a in np.mgrid[0:h, 0:w])
    ht = hit(n2w, w, h, d0, d1, fast, xs, ys)
    some = ht["g"]["some"]
    flat = ys * w + xs
    idx = flat[some]
    point = ht["point"][some]
    has, ridx, _, _ = _reproject(reproj, idx, w, h, mutation)
    f = _pick(has, _sub(gi_fields(res0), ridx), _zero_fields(len(idx)))
    f["conf"] = np.ones(len(idx), np.float32)
    c, dec = stored(f, fast, v1=point)
    return _result(idx, [_cand(np.ones(len(idx), bool), fold_und=~dec, **c)], {"fold": ~dec}, fields=f, point=point, has=has,
                   sky=flat[~some], reprojected=int(has.sum()), disoccluded=int((~has).sum()))


# ---- K14: temporal resampling ------------------------------------------------------------------------------------------------

def gi_temporal(n2w, n2w_prev, w, h, gb, gb_prev, reproj, res_cur, res_prev, seed, frame, fast, inline=False, mutation=None,
                rows=None):
    """K14 gi_temporal_resampling::main for every pixel (or those of `rows`).  res_cur: gi_reservoirs[1] as K13 left it; res_prev:
    gi_reservoirs[2] as K11 left it, or gi_reservoirs[0] for the inline form (ST_OPT_FUSED_PASSES on tracing frames), where K11 is
    composed in: the rhs is K11's reservoir with its normal through one more round trip, as the store / load through memory did.
      * lhs: gi_reservoirs[1] where got_sample (tracing frames: frame even and the checkerboard of frame / 2; validation frames:
        the checkerboard of frame), else the default reservoir.
      * rhs: where the reprojection exists, with confidence 1 and M clamped at 128; on validation frames, where lhs and rhs are
        nonempty and the rhs sample exists, the radiance-distance test and the lhs's radiance, v2 and normal; its hit is rebuilt
        with the previous camera from the previous G-buffer at round() of the reprojection.
      * tracing: Mis::gi_temporal (jacobian 1), two updates, M = lhs M + mis M, confidence 1, norm_mis.
      * validation: merge(rhs, rhs pdf), confidence of the rhs (0 where nothing reprojects), norm_avg.
      * pdf = the pdf taken, v1 = the hit point, w clamped at 5; sky pixels store the default reservoir."""
    tracing = tracing_frame(frame)
    ys, xs = (a.reshape(-1) for a in np.mgrid[0:h, 0:w])
    if rows is not None:
        keep = np.isin(ys, rows)
        xs, ys = xs[keep], ys[keep]
    flat = ys * w + xs
    lh_all = hit(n2w, w, h, gb[0], gb[1], fast, xs, ys)
    some = lh_all["g"]["some"]
    idx = flat[some]
    n = len(idx)
    xs, ys = xs[some], ys[some]
    lh = {k: (v[some] if not isinstance(v, dict) else {kk: vv[some] for kk, vv in v.items()}) for k, v in lh_all.items()}
    z = lambda a: Num(np.asarray(a, np.float64), 0.0, fast)
    zero = z(np.zeros(n))
    und = {}
    # lhs
    ph = frame if (mutation == "k14_phase_frame" or not tracing) else frame // 2
    got = (xs % 2) == (ph + ys) % 2
    if tracing:
        got &= frame % 2 == 0
    lhs = _pick(got, _sub(gi_fields(res_cur), idx), _zero_fields(n))
    lenc, ldec = oct_roundtrip(lhs["enc"], fast)
    # rhs
    has, ridx, rx, ry = _reproject(reproj, idx, w, h)
    k11 = _sub(gi_fields(res_prev), ridx if inline else idx)
    rhs = _pick(has, k11, _zero_fields(n))
    if inline:
        first, dec0 = oct_roundtrip(k11["enc"], fast)
        renc_src, dec0 = pick_enc(has, first, nan_enc(n, fast)), dec0 | ~has
    else:
        renc_src, dec0 = rhs["enc"], np.ones(n, bool)
    rhs["conf"] = np.where(has, 1.0, 0.0).astype(np.float32)
    m_clamp = 64.0 if mutation == "k14_m64" else M_CLAMP
    m_clamped = has & (rhs["m"] > m_clamp)
    rhs["m"] = np.minimum(rhs["m"], np.float32(m_clamp))
    renc, rdec = oct_roundtrip(renc_src, fast)
    rdec &= dec0
    conf_alt = np.zeros(n, bool)      # pixels whose rhs confidence may be 0 or 1
    reset = near = np.zeros(n, bool)
    if not tracing:
        cond = has & (lhs["m"] != 0) & (rhs["m"] != 0) & exists(rhs["v2"])
        dvec = z(lhs["rad"]) - z(rhs["rad"])
        d = dot3(dvec, dvec) if mutation == "k14_distance_squared" else dot3(dvec, dvec).sqrt()
        margin = d.v - DISTANCE
        dec = (np.abs(margin) > d.e) | (d.e == 0)
        und["distance"] = cond & ~dec
        conf_alt = cond & ~dec
        reset = cond & dec & (margin > 0)
        near = cond & (np.abs(margin) <= 1e-5)
        rhs["conf"] = np.where(reset, 0.0, rhs["conf"]).astype(np.float32)
        for k in ("rad", "v2"):
            rhs[k] = np.where(cond[:, None], lhs[k], rhs[k])
        renc = pick_enc(cond, lenc, renc)
        rdec = np.where(cond, ldec, rdec)
    # the rhs hit: the previous camera and the previous G-buffer at round() of the reprojection
    rh = hit(n2w_prev, w, h, gb_prev[0], gb_prev[1], fast, np.where(has, rx, 0), np.where(has, ry, 0))
    rhs_some = has & (rhs["m"] != 0) & rh["g"]["some"]
    rng = WhiteNoise(seed, xs, ys)
    cands = []
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        if tracing:
            use_lr = (lhs["m"] > 0) & rhs_some
            use_rl = rhs["m"] > 0
            p_lr, u1 = gi_pdf(lhs["rad"], lhs["v2"], rh)
            p_rl, u2 = gi_pdf(rhs["rad"], rhs["v2"], lh)
            lhs_rhs_pdf, rhs_lhs_pdf = where(use_lr, p_lr, zero), where(use_rl, p_rl, zero)
            und["specular"] = (u1 & use_lr) | (u2 & use_rl)
            lm, rm = z(lhs["m"]), z(rhs["m"])
            mis_m, lhs_mis, rhs_mis = _mis_eval(lm, rm, z(lhs["pdf"]), lhs_rhs_pdf, rhs_lhs_pdf, z(rhs["pdf"]))
            und["mis q0"] = (lhs_rhs_pdf.e > 0) & (lhs_rhs_pdf.v <= lhs_rhs_pdf.e) & (rhs["m"] > 0)
            m_out = lm + mis_m
            m_out = Num(m_out.v, np.where(und["mis q0"], np.inf, m_out.e), fast)
            wl = (lhs_mis * z(lhs["pdf"])) * z(lhs["w"])
            wr = (rhs_mis * rhs_lhs_pdf) * z(rhs["w"])
            W1 = zero + wl
            W2 = W1 + wr
            acc1, dec1 = _decide(rng.sample(), W1, wl)
            acc2, dec2 = _decide(rng.sample(), W2, wr)
            und["update"] = ~(dec1 & dec2)
            und["unbounded"] = ~np.isfinite(m_out.e) | ~np.isfinite(lhs_rhs_pdf.e) | ~np.isfinite(rhs_lhs_pdf.e)
            for a1 in (False, True):
                for a2 in (False, True):
                    allowed = np.where(dec1, acc1 == a1, True) & np.where(dec2, acc2 == a2, True)
                    if a2:
                        src, pdf, enc, fdec = rhs, rhs_lhs_pdf, renc, rdec
                    elif a1:
                        src, pdf, enc, fdec = lhs, z(lhs["pdf"]), lenc, ldec
                    else:
                        src, pdf, enc, fdec = _zero_fields(n), zero, nan_enc(n, fast), np.ones(n, bool)
                    cands.append(_temporal_cand(allowed, src, enc, fdec, pdf, W2, Num(np.ones(n), 0.0, fast), m_out,
                                                np.ones(n, np.float32), lh["point"], fast, mutation))
        else:
            merged = rhs["m"] > 0
            f32 = np.float32
            m32 = np.where(merged, (f32(0) + (rhs["m"] - f32(1))) + f32(1), f32(0)).astype(f32)
            weight = where(merged, (z(rhs["w"]) * z(rhs["m"])) * z(rhs["pdf"]), zero)
            W = zero + weight
            acc, dec = _decide(rng.sample(), W, weight)
            dec |= ~merged
            acc &= merged
            und["update"] = ~dec
            den = z(m32) if mutation != "k14_norm_mis_validation" else Num(np.ones(n), 0.0, fast)
            for a in (False, True):
                allowed = np.where(dec, acc == a, True) & (merged | (not a))
                if a:
                    src, pdf, enc, fdec = rhs, z(rhs["pdf"]), renc, rdec
                else:
                    src, pdf, enc, fdec = _zero_fields(n), zero, nan_enc(n, fast), np.ones(n, bool)
                for conf in (0.0, 1.0):
                    al = allowed & np.where(conf_alt, True, rhs["conf"] == conf)
                    cands.append(_temporal_cand(al, src, enc, fdec, pdf, W, den, z(m32), np.full(n, conf, np.float32), lh["point"],
                                                fast, mutation))
    und["fold"] = np.zeros(n, bool)
    for c in cands:
        und["fold"] |= c["allowed"] & c["fold_und"]
    skip = und.get("specular", np.zeros(n, bool))
    sky = flat[~some]
    return _result(idx, cands, und, skip, sky=sky, reprojected=int(has.sum()), disoccluded=int((~has).sum()),
                   conf_reset=int(reset.sum()), near_threshold=int(near.sum()), m_clamped=int(m_clamped.sum()), got=int(got.sum()))


def _temporal_cand(allowed, src, enc, fdec, pdf, W, den, m, conf, point, fast, mutation):
    """One K14 / K17 outcome: the sample of `src`, w = norm(W, pdf, 1, den) (reservoir.rs:63-71) clamped at 5."""
    n = len(allowed)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        d = pdf * den
        wn = W / d
    exact0 = (d.v == 0) & (d.e == 0)
    firm = np.abs(d.v) > d.e      # the f32 denominator is certainly nonzero
    w = Num(np.where(exact0 | ~firm, 0.0, wn.v), np.where(exact0, 0.0, np.where(firm, wn.e, np.inf)), fast)
    if mutation != "no_w_clamp":
        w = w.minimum(W_CLAMP)
    return _cand(allowed, src["rad"], m, point, w, src["v2"], pdf, enc, conf, src["rng"], fold_und=~fdec)


def temporal_sky(got, r, what):
    """K14's sky pixels hold the default reservoir: every word 0 but the normal, NaN."""
    g = np.asarray(got, np.float32).reshape(-1, 16)[r["sky"]]
    assert (g[:, [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 14, 15]].view(np.uint32) == 0).all() and np.isnan(g[:, 12:14]).all(), \
        f"{what}: a sky pixel does not hold the default reservoir"


# ---- K17: spatial merge ------------------------------------------------------------------------------------------------------

def gi_spatial_sample(res_in, d2, seed, frame, w, h, fast, mutation=None):
    """K17 gi_spatial_resampling::sample on every pair of the half-width grid.  d2: the (H, W, 4) texels K16 left (texel a: lhs-rhs
    visibility, rhs_idx + 1, jacobian; texel b: rhs-lhs visibility, lhs_rhs_pdf, rhs_lhs_pdf), exact inputs; a texel past the
    screen reads zero.  Mis::eval with the texel's jacobian, the rhs weight times the jacobian, M = lhs M + mis M, confidence 1,
    v1 from the lhs, norm_mis and the w clamp; no merge (rhs_idx 0, or past the frame: the kernel's guard) passes the lhs through.
    The other pixel of the pair is copied where both are on the screen.  Returns the restatement, `copies` and `written`."""
    npx = w * h
    res = gi_fields(res_in)
    d2 = np.asarray(d2, np.float32).reshape(h, w, 4)
    gx, gy, lx, ox = half_grid_pairs(w, h, frame)
    on = lx < w
    copies = (gy * w + ox)[on & (ox < w)]
    gx, gy, lx = gx[on], gy[on], lx[on]
    lidx = gy * w + lx
    n = len(lidx)
    ax, bx = gx * 2, gx * 2 + 1
    tz = np.zeros((n, 4), np.float32)
    ta = np.where((ax < w)[:, None], d2[gy, np.minimum(ax, w - 1)], tz)
    tb = np.where((bx < w)[:, None], d2[gy, np.minimum(bx, w - 1)], tz)
    rhs_idx = ta[:, 1].view(np.uint32).astype(np.int64)
    merge = (rhs_idx > 0) & (rhs_idx - 1 < npx)
    lhs, rhs = _sub(res, lidx), _sub(res, np.where(merge, rhs_idx - 1, 0))
    z = lambda a: Num(np.asarray(a, np.float64), 0.0, fast)
    jac = z(ta[:, 2])
    lenc, ldec = oct_roundtrip(lhs["enc"], fast)
    renc, rdec = oct_roundtrip(rhs["enc"], fast)
    cands = []
    und = {}
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        lhs_rhs_pdf = z(tb[:, 1]) * z(ta[:, 0])
        rhs_lhs_pdf = z(tb[:, 2]) * z(tb[:, 0])
        lm, rm = z(lhs["m"]), z(rhs["m"])
        mis_m, lhs_mis, rhs_mis = _mis_eval(lm, rm, z(lhs["pdf"]), lhs_rhs_pdf, rhs_lhs_pdf, z(rhs["pdf"]), rhs_jacobian=jac)
        wl = (lhs_mis * z(lhs["pdf"])) * z(lhs["w"])
        wr = (rhs_mis * rhs_lhs_pdf) * z(rhs["w"])
        if mutation != "k17_no_jacobian":
            wr = wr * jac
        rng = WhiteNoise(seed, lx, gy)
        W1 = z(np.zeros(n)) + wl
        W2 = W1 + wr
        acc1, dec1 = _decide(rng.sample(), W1, wl)
        acc2, dec2 = _decide(rng.sample(), W2, wr)
        m_out = lm + mis_m
        und["update"] = merge & ~(dec1 & dec2)
        und["unbounded"] = merge & ~np.isfinite(m_out.e)
        one = Num(np.ones(n), 0.0, fast)
        for a1 in (False, True):
            for a2 in (False, True):
                allowed = merge & np.where(dec1, acc1 == a1, True) & np.where(dec2, acc2 == a2, True)
                if a2:
                    src, pdf, enc, fdec = rhs, rhs_lhs_pdf, renc, rdec
                elif a1:
                    src, pdf, enc, fdec = lhs, z(lhs["pdf"]), lenc, ldec
                else:
                    src, pdf, enc, fdec = _zero_fields(n), z(np.zeros(n)), nan_enc(n, fast), np.ones(n, bool)
                v1 = rhs["v1"] if (mutation == "k17_rhs_v1" and a2) else lhs["v1"]
                cands.append(_temporal_cand(allowed, src, enc, fdec, pdf, W2, one, m_out, np.ones(n, np.float32), v1, fast, mutation))
    c, dec = stored(lhs, fast)
    cands.append(_cand(~merge, fold_und=~dec, **c))
    und["fold"] = np.zeros(n, bool)
    for c in cands:
        und["fold"] |= c["allowed"] & c["fold_und"]
    return _result(lidx, cands, und, copies=copies, merged=int(merge.sum()), passed=int((~merge).sum()),
                   written=np.concatenate([lidx, copies]))


def check_copies(got, res_in, copies, fast, what):
    """K17's copies of the other pixel of each pair (and K19's copy into gi_reservoirs[0]): the reservoir as read, its normal through
    the round trip.  Returns (largest ratio, undecided folds)."""
    f = _sub(gi_fields(res_in), copies)
    c, dec = stored(f, fast)
    r = _result(copies, [_cand(np.ones(len(copies), bool), fold_und=~dec, **c)], {"fold": ~dec})
    return check_gi(got, r, what), r["undecided"]["fold"]


# ---- K19: resolving ----------------------------------------------------------------------------------------------------------

def gi_resolving(n2w, w, h, d0, d1, res0, fast, mutation=None):
    """K19 gi_resolving::main for every pixel: at a surface w cosine radiance of gi_reservoirs[0]'s entry, times (1 - metallic) / pi
    for the diffuse and the specular BRDF (the true base colour) for the specular output, with its confidence; on the sky zero with
    confidence 1.  Returns dict(diff, spec (Num (H, W, 3)), conf (H, W), some, undecided (specular early-out))."""
    ht = hit(n2w, w, h, d0, d1, fast)
    some = ht["g"]["some"]
    f = gi_fields(res0)
    z = lambda a: Num(np.asarray(a, np.float64).reshape(h, w, *np.shape(a)[1:]), 0.0, fast)
    v2 = f["v2"].reshape(h, w, 3)
    cos = gi_cosine(v2, ht)
    rad = (z(f["w"]) * cos).x3() * z(f["rad"])
    met = ht["g"]["metallic"]
    brdf = (1.0 / Num(np.full(met.v.shape, PI), 0.0, fast)) if mutation == "k19_no_metallic" else (1.0 - met) / PI
    diff = rad * brdf.x3()
    sb, und = specular(ht["g"], gi_dir(v2, ht["point"]), -ht["dir"])
    spec = rad * sb
    return dict(diff=diff, spec=spec, conf=f["conf"].reshape(h, w).astype(np.float64), some=some, undecided=und & some)


def check_resolving(diff, spec, r, what, check_within):
    """K19's two outputs against the restatement.  Returns (ratio, undecided specular, bounds)."""
    some = r["some"]
    diff = np.asarray(diff, np.float32); spec = np.asarray(spec, np.float32)
    assert (diff[..., 3][some] == r["conf"][some]).all() and (spec[..., 3][some] == r["conf"][some]).all(), f"{what}: confidence"
    assert (diff[..., 3][~some] == 1).all() and (spec[..., 3][~some] == 1).all(), f"{what}: sky confidence"
    assert (diff[..., :3][~some] == 0).all() and (spec[..., :3][~some] == 0).all(), f"{what}: sky radiance"
    ratio = check_within(diff[..., :3][some], r["diff"].v[some], r["diff"].e[some], f"{what} diffuse")
    und = r["undecided"]
    took_zero = und[..., None] & (spec[..., :3] == 0)
    want = np.where(took_zero, 0.0, r["spec"].v)
    bound = np.where(took_zero, 0.0, r["spec"].e)
    ratio = max(ratio, check_within(spec[..., :3][some], want[some], bound[some], f"{what} specular"))
    return ratio, int(und.sum())
