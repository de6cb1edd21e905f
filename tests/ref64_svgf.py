"""Float64 restatement of the SVGF denoiser, frame composition and the Rgba8UnormSrgb store, with a per-pixel error bound.

Written from the reference's definitions (paths relative to the reference tree), not from the CUDA kernels or the oracle:
  * K20 `frame_denoising::reproject`          strolle-shaders/src/frame_denoising.rs:3-78
  * K21 `frame_denoising::estimate_variance`  strolle-shaders/src/frame_denoising.rs:80-217
  * K22 `frame_denoising::wavelet`            strolle-shaders/src/frame_denoising.rs:219-361, `sample_weight` :363-392
  * composition `frame_composition::fs`       strolle-shaders/src/frame_composition.rs:18-82
  * `BilinearFilter`                          strolle-gpu/src/utils/bilinear_filter.rs:25-108
  * `Reprojection`                            strolle-gpu/src/reprojection.rs:13-55
  * `Surface` / `SurfaceMap`                  strolle-gpu/src/surface.rs:14-17, :60-68; `Normal::decode` strolle-gpu/src/normal.rs
  * `BlueNoise`                               strolle-gpu/src/noise/blue.rs:15-27
  * luma                                      strolle-gpu/src/utils/vec3_ext.rs (`luma`: dot with (0.2126, 0.7152, 0.0722))
  * `lerp`                                    strolle-gpu/src/utils.rs:23-31 (`a + (b - a) * t.clamp(0, 1)`)
  * `GBufferEntry::unpack`                    strolle-gpu/src/gbuffer.rs:19-57, `to_bytes` strolle-gpu/src/utils/u32_ext.rs:14-25
  * Rgba8UnormSrgb                            strolle/src/camera.rs:180 (the viewport format); IEC 61966-2-1 encoding, clamp to
                                              [0, 1], round to nearest; NaN converts to 0 (Vulkan / D3D float -> UNORM rules)

Semantics that matter at the edges:
  * `Camera::contains` (strolle-gpu/src/camera.rs:116-132) rejects taps outside the frame; storage reads outside the frame return 0.
    `BilinearFilter::from_reprojection` only tests `p.x >= 0 && p.y >= 0`, so a corner at x = w (ceil of a fractional position on
    the last column) is read as 0 with weight 1.
  * sky means `depth == 0` (surface.rs:15-17).
  * glam 0.24: `fract` is `x - floor(x)`, `round` rounds half away from zero, `as_ivec2` / `as i32` truncate (saturating), and
    `as_uvec2` saturates negatives to 0.
  * K21's window is quirk C-3: row -2 spans x in [-2, 2], rows -1..2 span x in [-3, 2] (frame_denoising.rs:128-190).
  * K21 picks the moment path from the DI history alone (`center_di_moment.x >= 4.0`, frame_denoising.rs:122) for both signals.
  * History is capped at 16 (frame_denoising.rs:56); variance is clamped with `max(0)` (:207-208).
  * A sky centre in the wavelet writes DI through and leaves the GI output untouched (frame_denoising.rs:248-254).
  * jitter = trunc((bnoise.zw - 0.5) * (stride - 1) * 0.5) with the blue noise read at ((x + 71 f) mod 256, (y + 11 f) mod 256);
    strength = 1 + iteration, stride = 2^iteration (strolle/src/camera_controller/passes/frame_denoising.rs:185-186).

Discrete decisions.  The depth cut-off `diff >= leeway` is evaluated on the f32 values leeway = depth * (0.33f / strength) (resp.
depth * 0.2f in K21) and diff = |a - b|: each is one correctly rounded f32 operation and both tiers compute them the same way; the
ramp 1 - diff / leeway is then f64.  Every other predicate is exact on the f32 inputs (`confidence > 0`, `sample.w > 0`,
`history >= 4`, `is_exact`, floor / ceil of the previous position, sky).  The jitter is computed in f64: with k the blue-noise byte,
(k/255 - 1/2)(S - 1)/2 = (2k - 255)(S - 1)/1020 and 2k - 255 is odd, so for S = 2, 4, 8, 16 the value is never an integer (the
f32 evaluation cannot truncate differently: its distance to the nearest integer is >= 1/1020) and for S = 1 it is exactly 0.

Error bound, per output value and per tier (u = 2^-24, the f32 unit roundoff; gamma_n = n u / (1 - n u)).  Every function takes the
absolute error bound of its inputs (0 for buffers read from the device, the previous stage's bound when stages are chained) and
returns the bound of its outputs against the f32 evaluation:

  luma      l = 0.2126 r + 0.7152 g + 0.0722 b: two products and two sums (strict) or an FMA chain (fast):
            dl <= gamma_3 sum|c_i x_i| + sum c_i dx_i.  The fast tier flushes denormals: + FLT_MIN.
  sqrt      strict: correctly rounded, u sqrt(l); fast: sqrt.approx.ftz.f32, relative error <= 2^-23 (PTX ISA), and a denormal input
            flushes to 0, which is an absolute error <= sqrt(FLT_MIN).  Input error dl propagates as min(dl / (2 sqrt l), sqrt dl).
  exp(-x)   strict: Cephes expf, relative error <= EXP_REL (asserted through `oracle.math`, which is bit-identical to the device);
            fast: ex2.approx.ftz.f32 of x * -log2(e): relative error <= 2^-22 (PTX ISA gives 2^-22.5) plus the rounding of the
            scaled argument, 2 u x.  Argument error dx moves the result by the factor e^dx - 1.
  luma weight argument x = |sqrt(lc) - sqrt(ls)| sigma:  dx <= sigma (d sqrt lc + d sqrt ls) + |sqrt lc - sqrt ls| d sigma + 2 u x.
            The sqrt error enters as sigma (sqrt lc + sqrt ls) times the relative sqrt error.
  sigma     K22: lerp(2.5, 0.5, sqrt var) / lerp(1, 0, sqrt var); clamp is 1-Lipschitz, so d sigma <= 2 d sqrt var (DI),
            d sqrt var (GI), plus 2 u (|b - a| t + |sigma|) for the lerp's two roundings.
  depth     1 - diff / leeway = 1 - q: strict u q + u dw (division and subtraction); fast fma(-diff, rcp(leeway), 1): 2^-23 q + u dw.
  normal    d = n_c . n_s of two normals decoded in f32 (each component within NORMAL_DECODE_ERR of the f64 decode, asserted against
            surface_nd on the device): dd <= 2 sqrt(3) NORMAL_DECODE_ERR + gamma_3.  normal^64 is six squarings, each doubling
            the relative error and adding u: d(nw) <= 64 (d + dd)^63 dd + 64 u nw.
  weight    w = exp * dw * nw, two products: dw_i <= w (e^dx - 1 + exp error + 2 u) + exp nw d(dw) + exp dw d(nw) (+ FLT_MIN fast).
  average   m = sum w_i v_i / W: a weight error moves it by sum dw_i |v_i - m| / W (exact to first order); input errors by
            sum w_i dv_i / W; accumulation of n terms, products and the division by gamma_(2n+3) sum w_i |v_i| / W; the fast
            tier's rcp.approx adds 2^-23 |m|.  W is replaced by W - sum dw_i in the denominators.
  variance  K22 out var = sum w_i^2 v_i / W^2: (sum 2 w_i dw_i |v_i| + w_i^2 dv_i) / W^2 + 2 var sum dw_i / W + rounding as above.
            K21 window: var = 4 |m2 - m1^2|, dvar = 4 (dm2 + 2 |m1| dm1 + u m1^2 + u |m2 - m1^2|).
            K21 moments: var = m.z - m.y^2, dvar = dm.z + 2 |m.y| dm.y + u m.y^2 + u |var|.
  K20       bilinear history: weights are products of (1 - fract) terms (two roundings each), summed (three) and divided once:
            <= 12 u sum w_i |s_i| / W; lerp(a, b, t): u (2 |b - a| t + |out|) + (1 - t) da + t db + |b - a| dt;
            alpha = 1 / min(h + 1, 16): d alpha <= alpha (dh / h + u) with dh = d(history) + u h.
  compose   emissive + (dd + gd) * base + ds + gs: gamma_5 on the magnitudes plus |dd + gd| base POW22_REL, base = (b/255)^2.2 with
            Cephes powf (POW22_REL asserted on all 256 bytes) and the division's rounding times 2.2.  Mode 6: u |c / w|.
  sRGB      f32 constants 12.92f, 1.055f, 0.055f, 1/2.4f differ from the decimal ones by their (exactly computed) representation
            error; powf within POW_INV24_REL; t = e * 255 + 0.5 adds two roundings.  The byte may differ by 1 only where the f64 value
            of t is within its bound of an integer.

The bound is a first-order bound with every rounding counted once; all terms are evaluated per pixel in float64.
"""
import numpy as np

U = 2.0 ** -24                 # f32 unit roundoff (round to nearest)
ULP_REL = 2.0 ** -23           # one ulp, relative to the value
FLT_MIN = 2.0 ** -126
TINY = 2.0 ** -140             # absolute slack for results in the f32 denormal range (strict tier keeps denormals)

EXP_REL = 1.0 * ULP_REL        # Cephes expf on [-87, 0]                       (test_ref64_constants)
POW22_REL = 20.0 * ULP_REL     # Cephes powf(b / 255, 2.2) over the 256 bytes    (test_ref64_constants)
POW_INV24_REL = 4.0 * ULP_REL  # Cephes powf(x, 1/2.4f) on [0.0031308, 1]        (test_ref64_constants)
NORMAL_DECODE_ERR = 8.0 * U    # |f32 octahedral decode - f64 decode| per component (surface_nd check on the device)

EX2_REL = 2.0 ** -22           # ex2.approx.ftz.f32   (PTX ISA: max relative error 2^-22.5)
SQRT_REL = 2.0 ** -23          # sqrt.approx.ftz.f32  (PTX ISA: max relative error 2^-23)
RCP_REL = 2.0 ** -23           # rcp.approx.ftz.f32   (PTX ISA: max 1 ulp)

LUMA = np.array([0.2126, 0.7152, 0.0722], dtype=np.float32).astype(np.float64)   # the f32 constants the reference multiplies by

# K21 window, quirk C-3 (frame_denoising.rs:128-190)
VARIANCE_WINDOW = [(x, -2) for x in range(-2, 3)] + [(x, y) for y in range(-1, 3) for x in range(-3, 3)]


def gamma(n):
    return n * U / (1.0 - n * U)


def _f32(x):
    return float(np.float32(x))


# ---- small pieces ----------------------------------------------------------------------------------------------------------

def luma(c, dc=None, fast=False):
    """Luminance of c[..., :3] in f64 and its f32 evaluation bound."""
    c = np.asarray(c, dtype=np.float64)[..., :3]
    with np.errstate(invalid="ignore", over="ignore"):
        l = c @ LUMA
        d = gamma(3) * (np.abs(c) @ LUMA)
        if dc is not None:
            d = d + np.asarray(dc, dtype=np.float64)[..., :3] @ LUMA
    if fast:
        d = d + FLT_MIN
    return l, d


def sqrt_err(l, dl, fast):
    """|f32 sqrt(l~) - sqrt(l)| for |l~ - l| <= dl."""
    with np.errstate(invalid="ignore", divide="ignore"):
        s = np.sqrt(np.maximum(l, 0.0))
        prop = np.where(s > 0, np.minimum(dl / (2 * np.where(s > 0, s, 1.0)), np.sqrt(dl)), np.sqrt(dl))
        if fast:
            return SQRT_REL * s + np.sqrt(FLT_MIN) + prop
        return U * s + prop


def decode_normal(m):
    """Normal::decode (strolle-gpu/src/normal.rs) in f64 from the surface map's first two components."""
    m = np.asarray(m, dtype=np.float64)[..., 0:2] * 2.0 - 1.0
    n = np.stack([m[..., 0], m[..., 1], 1.0 - np.abs(m[..., 0]) - np.abs(m[..., 1])], -1)
    t = np.maximum(-n[..., 2], 0.0)
    n[..., 0] -= np.copysign(t, n[..., 0])
    n[..., 1] -= np.copysign(t, n[..., 1])
    with np.errstate(invalid="ignore", divide="ignore"):
        return n / np.linalg.norm(n, axis=-1, keepdims=True)


def surface(surface_map):
    """(normal f64 (H, W, 3), depth f32 (H, W)) of a surface map (SurfaceMap::get, surface.rs:60-68)."""
    s = np.asarray(surface_map, dtype=np.float32)
    return decode_normal(s), s[..., 2].copy()


def blue_noise_zw(bn, w, h, frame):
    """BlueNoise::second_sample (noise/blue.rs:15-27): the zw channels at ((x + 71 f) mod 256, (y + 11 f) mod 256), as k / 255."""
    ys, xs = np.mgrid[0:h, 0:w]
    ux, uy = (xs + 71 * frame) % 256, (ys + 11 * frame) % 256
    t = np.asarray(bn, dtype=np.uint8).reshape(256, 256, 4)[uy, ux]
    return t[..., 2].astype(np.int64), t[..., 3].astype(np.int64)


def jitter(bn, w, h, frame, stride):
    """((zw - 0.5) * (stride - 1) * 0.5).as_ivec2() in f64: never an integer for stride > 1 (module docstring)."""
    kz, kw = blue_noise_zw(bn, w, h, frame)
    jx = np.trunc((kz / 255.0 - 0.5) * (stride - 1) * 0.5).astype(np.int64)
    jy = np.trunc((kw / 255.0 - 0.5) * (stride - 1) * 0.5).astype(np.int64)
    return jx, jy


def _gather(a, sx, sy, ok):
    """a[sy, sx] where ok, 0 elsewhere (storage reads outside the frame return 0)."""
    h, w = a.shape[0], a.shape[1]
    v = a[np.clip(sy, 0, h - 1), np.clip(sx, 0, w - 1)]
    m = ok.reshape(ok.shape + (1,) * (v.ndim - ok.ndim))
    return np.where(m, v, 0)


def _round_half_away(x):
    return np.sign(x) * np.floor(np.abs(x) + 0.5)


def _as_i32(x):
    with np.errstate(invalid="ignore"):
        return np.where(np.isnan(x), 0, np.clip(np.trunc(x), -2.0 ** 31, 2.0 ** 31 - 1)).astype(np.int64)


def _lerp(a, b, t, da, db, dt):
    """lerp(a, b, t) = a + (b - a) * clamp(t, 0, 1) (utils.rs:23-31) and its f32 bound."""
    t = np.clip(t, 0.0, 1.0)
    out = a + (b - a) * t
    d = U * (2 * np.abs(b - a) * t + np.abs(out)) + (1 - t) * da + t * db + np.abs(b - a) * dt
    return out, d


def _depth_ramp(c_depth, s_depth, depth_sigma_f32, fast):
    """Depth weight of sample_weight (frame_denoising.rs:374-383): the cut-off on f32 leeway / diff, the ramp in f64."""
    c = np.asarray(c_depth, dtype=np.float32)
    s = np.asarray(s_depth, dtype=np.float32)
    leeway = (c * np.float32(depth_sigma_f32)).astype(np.float32)
    diff = np.abs(s - c).astype(np.float32)
    cut = ~(diff < leeway)          # diff >= leeway, and NaN compares false in both
    with np.errstate(invalid="ignore", divide="ignore"):
        q = np.where(cut, 0.0, diff.astype(np.float64) / np.where(cut, 1.0, leeway.astype(np.float64)))
    dw = np.where(cut, 0.0, 1.0 - q)
    ddw = np.where(cut, 0.0, (RCP_REL if fast else U) * q + U * dw)
    return dw, ddw


def _normal_weight(nc, ns, fast):
    d = np.sum(nc * ns, axis=-1)
    dd = 2 * np.sqrt(3.0) * NORMAL_DECODE_ERR + gamma(3)
    dp = np.maximum(d, 0.0)
    nw = dp ** 64
    dnw = 64 * np.minimum(dp + dd, 1.0 + dd) ** 63 * dd + 64 * U * nw
    return nw, dnw


def _exp_weight(x, dx, fast):
    """exp(-x) and the bound of its f32 evaluation given |x~ - x| <= dx."""
    with np.errstate(invalid="ignore", over="ignore"):
        e = np.exp(-x)
        rel = np.expm1(np.minimum(dx, 700.0)) + (EX2_REL + 2 * U * np.where(np.isfinite(x), x, 0.0) if fast else EXP_REL)
    return e, e * rel + (FLT_MIN if fast else TINY)


# ---- K20 -------------------------------------------------------------------------------------------------------------------

def reproject(sample, surface_map, reprojection, prev_colors, prev_moments, d_prev_colors=None, d_prev_moments=None):
    """frame_denoising::reproject for one signal.  Returns dict(color, moment, sky, b_color, b_moment); every array is (H, W, 4).
    At sky pixels `moment` is not written (its content is whatever the buffer held) and `color` is the sample itself.  The pass is
    strict IEEE arithmetic in both tiers, so there is one bound."""
    sample = np.asarray(sample, dtype=np.float32)
    h, w = sample.shape[:2]
    rp = np.asarray(reprojection, dtype=np.float32)
    pc = np.asarray(prev_colors, dtype=np.float64)
    pm = np.asarray(prev_moments, dtype=np.float64)
    dpc = np.zeros_like(pc) if d_prev_colors is None else np.asarray(d_prev_colors, dtype=np.float64)
    dpm = np.zeros_like(pm) if d_prev_moments is None else np.asarray(d_prev_moments, dtype=np.float64)
    sky = np.asarray(surface_map, dtype=np.float32)[..., 2] == 0
    s64 = sample.astype(np.float64)
    sl, dsl = luma(s64)
    valid = (rp[..., 2] > 0) & (sample[..., 3] > 0)
    px, py = rp[..., 0], rp[..., 1]
    fx, fy = (px - np.floor(px)).astype(np.float32), (py - np.floor(py)).astype(np.float32)
    exact = (fx * fx + fy * fy) == 0                    # length_squared in f32 (reprojection.rs:52-54)
    validity = rp[..., 3].view(np.uint32)

    # exact: prev_pos().round().as_uvec2()
    ex = np.clip(_round_half_away(px.astype(np.float64)), 0, None)
    ey = np.clip(_round_half_away(py.astype(np.float64)), 0, None)
    ex = np.where(np.isnan(ex), 0, np.minimum(ex, 2.0 ** 32)).astype(np.int64)
    ey = np.where(np.isnan(ey), 0, np.minimum(ey, 2.0 ** 32)).astype(np.int64)
    in_e = (ex < w) & (ey < h)
    hist_c, hist_m = _gather(pc, ex, ey, in_e), _gather(pm, ex, ey, in_e)
    dhist_c, dhist_m = _gather(dpc, ex, ey, in_e), _gather(dpm, ex, ey, in_e)

    # bilinear (bilinear_filter.rs:41-108)
    x0, x1 = _as_i32(np.floor(px.astype(np.float64))), _as_i32(np.ceil(px.astype(np.float64)))
    y0, y1 = _as_i32(np.floor(py.astype(np.float64))), _as_i32(np.ceil(py.astype(np.float64)))
    u_, v_ = fx.astype(np.float64), fy.astype(np.float64)
    corners = [(x0, y0, 1, (1 - u_) * (1 - v_)), (x1, y0, 2, u_ * (1 - v_)), (x0, y1, 4, (1 - u_) * v_), (x1, y1, 8, u_ * v_)]
    wsum = np.zeros((h, w))
    num_c, num_m = np.zeros((h, w, 4)), np.zeros((h, w, 4))
    abs_c, abs_m = np.zeros((h, w, 4)), np.zeros((h, w, 4))
    din_c, din_m = np.zeros((h, w, 4)), np.zeros((h, w, 4))
    for cx, cy, bit, f in corners:
        take = ((validity & bit) > 0) & (cx >= 0) & (cy >= 0)
        inside = take & (cx < w) & (cy < h)
        wt = np.where(take, f, 0.0)
        sc, sm = _gather(pc, cx, cy, inside), _gather(pm, cx, cy, inside)
        wsum += wt
        num_c += sc * wt[..., None]; num_m += sm * wt[..., None]
        abs_c += np.abs(sc) * wt[..., None]; abs_m += np.abs(sm) * wt[..., None]
        din_c += _gather(dpc, cx, cy, inside) * wt[..., None]; din_m += _gather(dpm, cx, cy, inside) * wt[..., None]
    nz = wsum != 0
    ws = np.where(nz, wsum, 1.0)[..., None]
    with np.errstate(invalid="ignore"):
        bil_c = np.where(nz[..., None], num_c / ws, 0.0)
        bil_m = np.where(nz[..., None], num_m / ws, 0.0)
        dbil_c = np.where(nz[..., None], 12 * U * abs_c / ws + din_c / ws, 0.0)
        dbil_m = np.where(nz[..., None], 12 * U * abs_m / ws + din_m / ws, 0.0)
    e3 = exact[..., None]
    prev_c = np.where(e3, hist_c, bil_c); dprev_c = np.where(e3, dhist_c, dbil_c)
    prev_m = np.where(e3, hist_m, bil_m); dprev_m = np.where(e3, dhist_m, dbil_m)

    hist = np.minimum(prev_m[..., 0] + 1.0, 16.0)
    dh = np.where(prev_m[..., 0] + 1.0 < 16.0, dprev_m[..., 0] + U * hist, dprev_m[..., 0])
    with np.errstate(divide="ignore", invalid="ignore"):
        alpha = 1.0 / hist
        dalpha = alpha * (dh / np.abs(hist) + U)
    color = np.zeros((h, w, 4)); dcolor = np.zeros((h, w, 4))
    with np.errstate(invalid="ignore", over="ignore"):
        for k in range(3):
            o, d = _lerp(prev_c[..., k], s64[..., k], alpha, dprev_c[..., k], 0.0, dalpha)
            color[..., k] = np.where(valid, o, s64[..., k]); dcolor[..., k] = np.where(valid, d, 0.0)
        m1, dm1 = _lerp(prev_m[..., 1], sl, alpha, dprev_m[..., 1], dsl, dalpha)
        sl2, dsl2 = sl * sl, 2 * np.abs(sl) * dsl + U * sl * sl
        m2, dm2 = _lerp(prev_m[..., 2], sl2, alpha, dprev_m[..., 2], dsl2, dalpha)
    moment = np.stack([np.where(valid, hist, 1.0), np.where(valid, m1, sl), np.where(valid, m2, sl2), np.zeros((h, w))], -1)
    dmoment = np.stack([np.where(valid, dh, 0.0), np.where(valid, dm1, dsl), np.where(valid, dm2, dsl2), np.zeros((h, w))], -1)
    color = np.where(sky[..., None], s64, color)
    dcolor = np.where(sky[..., None], 0.0, dcolor + TINY)
    dmoment = dmoment + TINY
    return dict(color=color, moment=moment, sky=sky, b_color=dcolor, b_moment=dmoment)


# ---- K21 -------------------------------------------------------------------------------------------------------------------

def _sqrt_luma(c, dc, fast):
    l, dl = luma(c, dc, fast)
    with np.errstate(invalid="ignore"):
        return l, dl, np.sqrt(l), sqrt_err(l, dl, fast)


def estimate_variance(surface_map, colors, moments, d_colors=None, d_moments=None, fast=False):
    """frame_denoising::estimate_variance.  `colors` / `moments` / `d_*` are dicts {"di": (H, W, 4), "gi": (H, W, 4)}.
    Returns dict {"di": out, "gi": out, "b_di": bound, "b_gi": bound, "sky": mask}."""
    normal, depth = surface(surface_map)
    h, w = depth.shape
    sky = depth == 0
    ys, xs = np.mgrid[0:h, 0:w]
    out = {"sky": sky}
    hist_ok = np.asarray(moments["di"], dtype=np.float32)[..., 0] >= 4.0
    taps = []
    for ox, oy in VARIANCE_WINDOW:
        sx, sy = xs + ox, ys + oy
        ok = (sx >= 0) & (sy >= 0) & (sx < w) & (sy < h)
        sdep = _gather(depth, sx, sy, ok)
        ok = ok & (sdep != 0)
        dw, ddw = _depth_ramp(depth, sdep, np.float32(0.2), fast)
        nw, dnw = _normal_weight(normal, _gather(normal, sx, sy, ok), fast)
        taps.append((sx, sy, ok, dw, ddw, nw, dnw))
    for sig in ("di", "gi"):
        c = np.asarray(colors[sig], dtype=np.float64)
        dc = np.zeros_like(c) if d_colors is None else np.asarray(d_colors[sig], dtype=np.float64)
        m = np.asarray(moments[sig], dtype=np.float64)
        dm = np.zeros_like(m) if d_moments is None else np.asarray(d_moments[sig], dtype=np.float64)
        with np.errstate(invalid="ignore", over="ignore"):
            var_m = m[..., 2] - m[..., 1] ** 2
            dvar_m = dm[..., 2] + 2 * np.abs(m[..., 1]) * dm[..., 1] + U * m[..., 1] ** 2 + U * np.abs(var_m)
        lc, dlc, sc, dsc = _sqrt_luma(c, dc, fast)
        S0 = np.zeros((h, w)); S1 = np.zeros((h, w)); S2 = np.zeros((h, w))
        A1 = np.zeros((h, w)); A2 = np.zeros((h, w)); DW = np.zeros((h, w))
        per_tap = []
        with np.errstate(invalid="ignore", over="ignore"):
            for sx, sy, ok, dw, ddw, nw, dnw in taps:
                ls, dls, ss, dss = _sqrt_luma(_gather(c, sx, sy, ok), _gather(dc, sx, sy, ok), fast)
                x = np.abs(sc - ss)
                dx = dsc + dss + 2 * U * x
                e, de = _exp_weight(x, dx, fast)
                wt = np.where(ok, e * dw * nw, 0.0)
                dwt = np.where(ok, de * dw * nw + e * ddw * nw + e * dw * dnw + 2 * U * wt, 0.0)
                S0 += wt; S1 += wt * ls; S2 += wt * ls * ls
                A1 += wt * np.abs(ls); A2 += wt * ls * ls; DW += dwt
                per_tap.append((wt, dwt, ls, dls))
            m1, m2 = S1 / S0, S2 / S0
            lo = np.maximum(S0 - DW, 0.5 * S0)
            E1 = np.zeros((h, w)); E2 = np.zeros((h, w))
            for wt, dwt, ls, dls in per_tap:
                E1 += dwt * np.abs(ls - m1) + wt * dls
                E2 += dwt * np.abs(ls * ls - m2) + wt * (2 * np.abs(ls) * dls + U * ls * ls)
            dm1 = E1 / lo + gamma(2 * 29 + 3) * A1 / S0
            dm2 = E2 / lo + gamma(2 * 29 + 3) * A2 / S0
            diff = m2 - m1 * m1
            var_w = np.abs(diff) * 4.0
            dvar_w = 4 * (dm2 + 2 * np.abs(m1) * dm1 + U * m1 * m1 + U * np.abs(diff))
            var = np.where(hist_ok, var_m, var_w)
            dvar = np.where(hist_ok, dvar_m, dvar_w)
            var_c = np.where(np.isnan(var), 0.0, np.maximum(var, 0.0))   # f32::max returns the operand that is not NaN
        res = np.concatenate([c[..., :3], var_c[..., None]], -1)
        b = np.concatenate([np.zeros(c[..., :3].shape) + dc[..., :3], (dvar + (FLT_MIN if fast else TINY))[..., None]], -1)
        out[sig] = np.where(sky[..., None], c, res)
        out["b_" + sig] = np.where(sky[..., None], dc, b)
    return out


# ---- K22 -------------------------------------------------------------------------------------------------------------------

def wavelet(surface_map, di_in, gi_in, iteration, frame, bn, d_di=None, d_gi=None, fast=False):
    """One à-trous iteration (frame_denoising::wavelet) with stride 2^iteration and strength 1 + iteration.
    Returns dict {"di", "gi", "b_di", "b_gi", "sky"}: at sky pixels "di" is the input and "gi" is NaN (not written)."""
    stride, strength = 2 ** iteration, np.float32(1 + iteration)
    normal, depth = surface(surface_map)
    h, w = depth.shape
    sky = depth == 0
    ys, xs = np.mgrid[0:h, 0:w]
    jx, jy = jitter(bn, w, h, frame, stride)
    depth_sigma = np.float32(0.33) / strength
    taps = []
    for oy in (-1, 0, 1):
        for ox in (-1, 0, 1):
            if ox == 0 and oy == 0:
                continue
            sx, sy = xs + jx + ox * stride, ys + jy + oy * stride
            ok = (sx >= 0) & (sy >= 0) & (sx < w) & (sy < h)
            sdep = _gather(depth, sx, sy, ok)
            ok = ok & (sdep != 0)
            dw, ddw = _depth_ramp(depth, sdep, depth_sigma, fast)
            nw, dnw = _normal_weight(normal, _gather(normal, sx, sy, ok), fast)
            taps.append((sx, sy, ok, dw, ddw, nw, dnw))
    out = {"sky": sky}
    for sig, arr, darr, (a, b) in (("di", di_in, d_di, (2.5, 0.5)), ("gi", gi_in, d_gi, (1.0, 0.0))):
        c = np.asarray(arr, dtype=np.float64)
        dc = np.zeros_like(c) if darr is None else np.asarray(darr, dtype=np.float64)
        with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
            lc, dlc, sc, dsc = _sqrt_luma(c, dc, fast)
            sv = np.sqrt(c[..., 3])
            dsv = sqrt_err(c[..., 3], dc[..., 3], fast)
            t = np.clip(sv, 0.0, 1.0)
            sigma = a + (b - a) * t
            dsigma = abs(b - a) * dsv + 2 * U * (abs(b - a) * t + np.abs(sigma))
            W = np.ones((h, w)); SC = c[..., :3].copy(); SV = c[..., 3].copy()
            AC = np.abs(c[..., :3]).copy(); AV = np.abs(c[..., 3]).copy()
            per_tap = []
            for sx, sy, ok, dw, ddw, nw, dnw in taps:
                s = _gather(c, sx, sy, ok); ds = _gather(dc, sx, sy, ok)
                ls, dls, ss, dss = _sqrt_luma(s, ds, fast)
                x = np.abs(sc - ss) * sigma
                dx = sigma * (dsc + dss) + np.abs(sc - ss) * dsigma + 2 * U * x
                e, de = _exp_weight(x, dx, fast)
                wt = e * dw * nw
                use = ok & (wt > 0)                       # `if sample_weight > 0.0` (NaN weights are skipped)
                wt = np.where(use, wt, 0.0)
                dwt = np.where(use | (ok & np.isfinite(x)), de * dw * nw + e * ddw * nw + e * dw * dnw + 2 * U * wt, 0.0)
                sq = np.where(use[..., None], s, 0.0)
                W += wt; SC += wt[..., None] * sq[..., :3]; SV += wt * wt * sq[..., 3]
                AC += wt[..., None] * np.abs(sq[..., :3]); AV += wt * wt * np.abs(sq[..., 3])
                per_tap.append((wt, dwt, sq, np.where(use[..., None], ds, 0.0), ok))
            oc = SC / W[..., None]
            ov = SV / (W * W)
            DW = sum(p[1] for p in per_tap)
            lo = np.maximum(W - DW, 0.5 * W)
            Ec = dc[..., :3].copy(); Ev = dc[..., 3].copy()
            Ew = np.zeros((h, w))
            for wt, dwt, sq, dsq, ok in per_tap:
                Ec += dwt[..., None] * np.abs(sq[..., :3] - oc) + wt[..., None] * dsq[..., :3]
                Ev += 2 * wt * dwt * np.abs(sq[..., 3]) + wt * wt * dsq[..., 3]
                Ew += dwt
            rnd = gamma(2 * 9 + 3)
            bc = Ec / lo[..., None] + rnd * AC / W[..., None]
            bv = Ev / (lo * lo) + 2 * np.abs(ov) * Ew / lo + rnd * AV / (W * W)
            if fast:
                bc = bc + (RCP_REL + U) * np.abs(oc) + FLT_MIN
                bv = bv + (2 * RCP_REL + 2 * U) * np.abs(ov) + FLT_MIN
            else:
                bc = bc + TINY
                bv = bv + TINY
        res = np.concatenate([oc, ov[..., None]], -1)
        bres = np.concatenate([bc, bv[..., None]], -1)
        if sig == "di":
            out["di"] = np.where(sky[..., None], c, res)
            out["b_di"] = np.where(sky[..., None], dc, bres)
        else:
            out["gi"] = np.where(sky[..., None], np.nan, res)
            out["b_gi"] = np.where(sky[..., None], 0.0, bres)
    return out


def wavelet_chain(surface_map, di_in, gi_in, iterations, frame, bn, d_di=None, d_gi=None, fast=False):
    """Several iterations in a row, each one's output (and bound) the next one's input.  GI at sky pixels is never read (sky
    centres only pass DI through, sky taps are skipped), so the unwritten values are carried as 0."""
    di, gi, bdi, bgi = di_in, gi_in, d_di, d_gi
    r = None
    for it in iterations:
        r = wavelet(surface_map, di, gi, it, frame, bn, bdi, bgi, fast)
        di, bdi = r["di"], r["b_di"]
        gi = np.where(r["sky"][..., None], 0.0, r["gi"])
        bgi = r["b_gi"]
    return r


# ---- composition -----------------------------------------------------------------------------------------------------------

def base_color(d1w):
    """GBufferEntry::unpack's base colour (gbuffer.rs:36-46): bytes of d1.w, little end first, (b / 255)^2.2 (alpha / 63)."""
    b = np.asarray(d1w, dtype=np.float32).view(np.uint32)
    by = np.stack([(b >> (8 * k)) & 0xFF for k in range(4)], -1).astype(np.float64)
    return (by / np.array([255.0, 255.0, 255.0, 63.0])) ** 2.2


def compose(mode, d0, d1, di_diff, gi_diff, di_spec, gi_spec, ref_colors, d_di=None, d_gi=None, fast=False):
    """frame_composition::fs: rgb in f64 (H, W, 3) and its bound; alpha is 1."""
    d0 = np.asarray(d0, dtype=np.float32); d1 = np.asarray(d1, dtype=np.float32)
    dd, gd = np.asarray(di_diff, np.float64)[..., :3], np.asarray(gi_diff, np.float64)[..., :3]
    ds, gs = np.asarray(di_spec, np.float64)[..., :3], np.asarray(gi_spec, np.float64)[..., :3]
    rc = np.asarray(ref_colors, np.float64)
    bdd = np.zeros_like(dd) if d_di is None else np.asarray(d_di, np.float64)[..., :3]
    bgd = np.zeros_like(gd) if d_gi is None else np.asarray(d_gi, np.float64)[..., :3]
    z = np.zeros_like(dd)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        if mode == 0:
            some = d0[..., 0] != 0                     # GBufferEntry::is_some: depth != 0 (gbuffer.rs:114-116)
            em = d1[..., :3].astype(np.float64)
            bc = base_color(d1[..., 3])[..., :3]
            s = dd + gd
            col = em + s * bc + ds + gs
            mag = np.abs(em) + np.abs(s) * bc + np.abs(ds) + np.abs(gs)
            b = gamma(5) * mag + np.abs(s) * bc * (POW22_REL + 2.2 * U) + (bdd + bgd) * bc + TINY
            return np.where(some[..., None], col, dd), np.where(some[..., None], b, bdd)
        if mode == 1:
            return dd, bdd
        if mode == 2:
            return ds, z
        if mode == 3:
            return gd, bgd
        if mode == 4:
            return gs, z
        if mode == 5:
            return rc[..., :3], z
        if mode == 6:
            v = rc[..., :3] / rc[..., 3:4]
            return v, U * np.abs(v) + TINY
    return z, z


# ---- Rgba8UnormSrgb --------------------------------------------------------------------------------------------------------

_C1292, _C1055, _C0055, _CEXP = 12.92, 1.055, 0.055, 1.0 / 2.4
_F1292, _F1055, _F0055 = _f32(12.92), _f32(1.055), _f32(0.055)
_FEXP = float(np.float32(1.0) / np.float32(2.4))
_FTHRESH = np.float32(0.0031308)


def srgb_encode(v):
    """The Rgba8UnormSrgb store of linear values v (any shape, f32): (expected byte, t, bound of t) where t = e * 255 + 0.5 in f64
    and the byte is floor(t); the f32 store may differ by one only where |t - round(t)| <= bound."""
    v = np.asarray(v, dtype=np.float32)
    x32 = np.where(np.isnan(v), np.float32(0), np.clip(v, np.float32(0), np.float32(1))).astype(np.float32)
    x = x32.astype(np.float64)
    lin = x32 <= _FTHRESH
    with np.errstate(divide="ignore", invalid="ignore"):
        p = x ** _CEXP
        e_lin = _C1292 * x
        e_pow = _C1055 * p - _C0055
        e = np.where(lin, e_lin, e_pow)
        de_lin = e_lin * (abs(_F1292 - _C1292) / _C1292 + U)
        lnx = np.where(x > 0, np.abs(np.log(np.where(x > 0, x, 1.0))), 0.0)
        de_pow = (_C1055 * p * (POW_INV24_REL + lnx * abs(_FEXP - _CEXP) + abs(_F1055 - _C1055) / _C1055 + U)
                  + abs(_F0055 - _C0055) + U * np.abs(e_pow))
    de = np.where(lin, de_lin, de_pow)
    e = np.clip(e, 0.0, 1.0)
    t = e * 255.0 + 0.5
    dt = 255.0 * de + U * 255.0 * e + U * t
    byte = np.clip(np.floor(t), 0, 255).astype(np.int64)
    return byte, t, dt
