"""Float64 restatement of the DI sampling (K5), the DI temporal resampling (K6), the DI spatial merge (K9) and DI resolving (K10), with
a per-value error bound for either arithmetic tier, and a check of the spatial visibility pass (K8) against the traversal.

Written from the reference's definitions (paths relative to the reference tree), not from the CUDA kernels or the oracle:
  * K5  `di_sampling::main`               strolle-shaders/src/di_sampling.rs:4-94; `EphemeralReservoir::build`
                                          strolle-gpu/src/reservoir/ephemeral.rs:14-55; `EphemeralSample::pdf` = `perc_luma` of the
                                          radiance, strolle-gpu/src/utils/vec3_ext.rs:56-58; `BlueNoise` strolle-gpu/src/noise/blue.rs
  * `Light::ray_bnoise`                   strolle-gpu/src/light.rs:217-239; glam 0.24 `any_orthonormal_pair` (Duff et al. 2017)
  * K6  `di_temporal_resampling::main`    strolle-shaders/src/di_temporal_resampling.rs:4-112
  * K7  `di_spatial_resampling::pick`     strolle-shaders/src/di_spatial_resampling.rs:4-147; `resolve_checkerboard_alt` strolle-gpu/src/utils.rs:37;
                                          `WhiteNoise::sample_disk` strolle-gpu/src/noise/white.rs:52-56; `Camera::contain`
                                          strolle-gpu/src/camera.rs:57-77; `DiSample::ray` strolle-gpu/src/reservoir/di.rs:119-123;
                                          `Normal::encode` strolle-gpu/src/normal.rs:9-23
  * K8  `di_spatial_resampling::trace`    strolle-shaders/src/di_spatial_resampling.rs:150-209
  * `Mis::di_temporal`                    strolle-gpu/src/reservoir/mis.rs:36-65
  * `DiSample::pdf` / `pdf_prev` / `pdf_ex`   strolle-gpu/src/reservoir/di.rs:95-117; `Light::contains` / slots / `rollback`
                                          strolle-gpu/src/light.rs:83-85, :107-141; `LightsView::get_prev` strolle-gpu/src/lights.rs:19-24
  * `Reprojection::prev_pos_round`        strolle-gpu/src/reprojection.rs:46-48; `Reservoir::clamp_m` strolle-gpu/src/reservoir.rs:55-57
  * K9  `di_spatial_resampling::sample`   strolle-shaders/src/di_spatial_resampling.rs:212-297
  * K10 `di_resolving::main`              strolle-shaders/src/di_resolving.rs:4-119
  * `Mis::eval`                           strolle-gpu/src/reservoir/mis.rs:96-145 (`m(q0, q1)` = (q1 / q0).min(1).powf(8).saturate())
  * `Reservoir::update` / `norm`          strolle-gpu/src/reservoir.rs:24-39, :63-79
  * `DiReservoir::read` / `write`         strolle-gpu/src/reservoir/di.rs:17-59 (m, w, pdf, bytes(occluded, confidence); point, id)
  * `Light::radiance`                     strolle-gpu/src/light.rs:143-207
  * `DiffuseBrdf::eval`, `SpecularBrdf::eval`, GGX terms   strolle-gpu/src/brdf.rs:20-24, :46-79, :162-186
  * `GBufferEntry::unpack`, `clamped_roughness`            strolle-gpu/src/gbuffer.rs:19-57, :118-120
  * `Camera::ray`                         strolle-gpu/src/camera.rs:80-93; `Camera::serialize` strolle/src/camera.rs:50-66
  * `Hit::new`                            strolle-gpu/src/hit.rs (point = origin + dir * (depth - 0.01))
  * `Normal::decode`                      strolle-gpu/src/normal.rs
  * `WhiteNoise`                          strolle-gpu/src/noise/white.rs (PCG hash, sample = u32 / 2^32)
  * glam 0.24: `angle_between` = acos_approx(dot / sqrt(|a|^2 |b|^2)), `reflect` = self - 2 dot(n, self) n, `normalize` = v * (1 / |v|),
    `project_point3` = (M v).xyz * (1 / w), `Mat4::inverse` by cofactors, `saturate` / `clamp` / `min` / `max` (SURVEY App. D).
  * per-dispatch seeds: dispatch_seed(base, frame, k) = pcg(base ^ (64 frame + k)), k = the pass id (K9: 5).

Arithmetic model.  The device evaluates the reference's f32 program; `Num` carries, per value, the f64 result of the same program and an
absolute bound on |f32 evaluation - f64 value| (u = 2^-24, the unit roundoff of round to nearest):
  a + b, a - b   e = ea + eb + u |r|.  An FMA contraction (the fast build, -fmad=true) rounds once where two roundings were counted,
                 so it is covered by the same term.
  a * b          e = |a| eb + |b| ea + ea eb + u |r|.
  a / b          e = (ea + |r| eb) / (|b| - eb) + rel |r|: rel = u (strict: correctly rounded); rel = 2^-22 in the fast build
                 (-prec-div=false: div.full.f32 is within 2 ulp, rcp.approx.f32 within 1 ulp, a product by a rounded reciprocal within
                 2 u).  |b| <= eb gives an infinite bound.
  sqrt a         |sqrt(a~) - sqrt(a)| <= min(ea / sqrt(a), sqrt(ea)), plus rel sqrt(a): u (strict) or 2^-23 (sqrt.approx.f32, PTX ISA).
                 1 / sqrt as a division of a square root also covers a fused rsqrt.approx.f32 (2^-22.9 < 2^-22 + 2^-23).
  min, max, clamp, saturate, |x|   1-Lipschitz: the input bound passes through; where the value is past a limit by more than its
                 bound the f32 result is that limit, exactly (bound 0).
  powf(x, k)     for k = 3, 5, 8 the reference's exponents are evaluated as the products x x x, (x^2)^2 x, ((x^2)^2)^2 in both tiers.
  Every rounding of a result in the f32 subnormal range adds 2^-149 (neither build flushes denormals).
Inputs read from device buffers are exact (e = 0).  The base colour is (b / 255)^2.2 from a 256-entry table the strict pow builds:
relative error POW22_REL + 2.2 u (tests/ref64_svgf.py, asserted on all bytes).  The camera matrix `ndc_to_world` is computed on the host
in f32 (Camera::serialize, glam's Mat4::inverse and Mat4 * Mat4), which is restated here operation for operation in f32, so it is exact.
`acos_approx` is glam's polynomial evaluated through `Num`; its sign branch (pi - r for v < 0) is continuous to 5e-8, added as slack.

Discrete decisions.  Each is evaluated on the f64 values with its bound:
  * `n.l <= 0 || n.v <= 0` in SpecularBrdf::eval: decided where |dot| > its bound; otherwise the pixel's specular term is *undecided*
    and the device may return 0 or the value.
  * `rng * W < weight` in Reservoir::update: the draw is exact (a u32 times 2^-32, rounded once to f32 and computed exactly here);
    decided where |rng W - weight| > rng eW + eweight + u rng W.  Both branches consume one draw, so an undecided update only doubles
    the candidate outcomes: every consistent combination is computed and the device's result must match one of them exactly in its
    discrete fields (light id, light point, occluded, confidence, pdf) and within the bound in its continuous ones (m, w).
    A product with an exactly zero factor is exactly zero; a comparison of exact values is decided.
  * `q0 <= 0`, `sum == 0`, `rhs_idx > 0`, `pdf * 1 == 0` and `lhs_rhs_vis == 0` act on values that are exact f32 inputs or exact
    products of them, so they are decided.
  * K6: `Light::contains(light_point)` in pdf_ex compares a rounded distance with the radius; where |d - R| is inside d's bound the
    pdf may be 0 or the value, and the pixel is counted as undecided and not compared.  The same holds for the specular early-out in
    any of K6's three pdfs.  `q0 <= 0` in m(q0, q1) acts on the recomputed lhs_rhs_pdf: where 0 < q0 <= its bound (or q0 = 0 with a
    nonzero bound) m is left unbounded and the pixel is counted, as is any pixel whose pdfs have no finite bound.  `round()` of the
    reprojection and the slot markers act on exact inputs.
  * K5: the selection.  Each of the min(light_count, 16) updates is an `rng * W < weight` decision, and W does not depend on which
    candidates were taken, so the consistent final selections are the last decided accept plus every undecided step after it (no
    selection at all when none was decided accepted).  The set is linear in the number of steps.  A selection's pdf = 0 (norm_avg's
    `denom == 0`) is decided only where the pdf is exactly 0 or certainly nonzero; otherwise w is left unbounded.
  * K5: `signum(light_dir.z)` in any_orthonormal_pair: decided where |z| exceeds its bound; otherwise the light point of either sign
    is accepted and the pixel is counted.  The occluded bit is compared with the traversal of the ray rebuilt in strict f32
    (`ray_bnoise_f32`), which the strict build must match on every ray and whose light point it must reproduce bit for bit.
  A quotient 0 / b of an exact zero by a divisor certainly nonzero is exactly zero (as a product with an exact zero factor is).
Visibility (Ray::intersect) is not restated: K9 takes it from the scratch texels, K10 from the occluded bit it stores, and K8's bit is
compared with the engine's any-hit traversal of the ray decoded from K7's texels (`oct_decode_f32`: the strict build's decode exactly).
"""
import numpy as np

from tests.ref64_svgf import U, POW22_REL

DIV_REL = 2.0 ** -22     # fast build: div.full.f32 (2 ulp), rcp.approx.f32 (1 ulp)
SQRT_REL_FAST = 2.0 ** -23   # sqrt.approx.f32 (PTX ISA)
SUB = 2.0 ** -149        # rounding of a subnormal result
PI = float(np.float32(np.pi))
ACOS_BRANCH = 5e-8
CLAMPED_ROUGHNESS_MIN = float(np.float32(np.float32(0.089) * np.float32(0.089)))
F32_EPS = float(np.finfo(np.float32).eps)


def _f32c(x):
    return float(np.float32(x))


# ---- running-error numbers --------------------------------------------------------------------------------------------------

class Num:
    """A float64 value array and an absolute bound on the f32 evaluation's distance from it (module docstring)."""
    __array_ufunc__ = None   # ndarray (op) Num defers to Num's reflected operators

    def __init__(self, v, e=0.0, fast=False):
        self.v = np.asarray(v, dtype=np.float64)
        e = np.asarray(e, dtype=np.float64)
        if e.shape != self.v.shape:
            e = np.broadcast_to(e, self.v.shape)
        self.e = np.where(np.isnan(e), np.inf, e)      # a bound lost to inf * 0 or inf - inf is no bound
        self.fast = fast

    def _n(self, x):
        return x if isinstance(x, Num) else Num(x, 0.0, self.fast)

    def __getitem__(self, k):
        return Num(self.v[k], self.e[k], self.fast)

    def col(self, i):
        return Num(self.v[..., i], self.e[..., i], self.fast)

    def x3(self):   # a scalar per pixel, broadcast against a vec3
        return Num(self.v[..., None], self.e[..., None], self.fast)

    @staticmethod
    def _sub(r, *input_bounds):
        """2^-149 wherever the f32 result may be a rounded subnormal: not for an exact zero computed from exact inputs."""
        m = r != 0
        for e in input_bounds:
            m = m | (e > 0)
        return np.where(m, SUB, 0.0)

    def __add__(self, o):
        o = self._n(o)
        with np.errstate(invalid="ignore", over="ignore"):
            r = self.v + o.v
            return Num(r, self.e + o.e + U * np.abs(r), self.fast)
    __radd__ = __add__

    def __sub__(self, o):
        o = self._n(o)
        with np.errstate(invalid="ignore", over="ignore"):
            r = self.v - o.v
            return Num(r, self.e + o.e + U * np.abs(r), self.fast)

    def __rsub__(self, o):
        return self._n(o) - self

    def __neg__(self):
        return Num(-self.v, self.e, self.fast)

    def __mul__(self, o):
        o = self._n(o)
        with np.errstate(invalid="ignore", over="ignore"):
            r = self.v * o.v
            e = np.abs(self.v) * o.e + np.abs(o.v) * self.e + self.e * o.e + U * np.abs(r) + self._sub(r, self.e, o.e)
            exact_zero = ((self.v == 0) & (self.e == 0) & np.isfinite(o.v)) | ((o.v == 0) & (o.e == 0) & np.isfinite(self.v))
            return Num(r, np.where(exact_zero, 0.0, e), self.fast)
    __rmul__ = __mul__

    def __truediv__(self, o):
        o = self._n(o)
        rel = DIV_REL if self.fast else U
        with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
            r = self.v / o.v
            lo = np.abs(o.v) - o.e
            e = np.where(lo > 0, (self.e + np.abs(r) * o.e) / np.where(lo > 0, lo, 1.0), np.inf) + rel * np.abs(r)
            exact_zero = (self.v == 0) & (self.e == 0) & (lo > 0) & np.isfinite(o.v)     # 0 / b is 0 for any f32 b != 0
            return Num(r, np.where(exact_zero, 0.0, e + self._sub(r, self.e, o.e)), self.fast)

    def __rtruediv__(self, o):
        return self._n(o) / self

    def sqrt(self):
        rel = SQRT_REL_FAST if self.fast else U
        with np.errstate(invalid="ignore", divide="ignore"):
            s = np.sqrt(np.maximum(self.v, 0.0))
            prop = np.where(s > 0, np.minimum(self.e / np.where(s > 0, s, 1.0), np.sqrt(self.e)), np.sqrt(self.e))
            return Num(s, prop + rel * s + self._sub(s, self.e), self.fast)

    def clip(self, lo, hi):
        """Where the f32 value is certainly past a limit (by more than its bound) the result is that limit, exactly."""
        with np.errstate(invalid="ignore"):
            pinned = (self.v < lo - self.e) | (self.v > hi + self.e)
        return Num(np.clip(self.v, lo, hi), np.where(pinned, 0.0, self.e), self.fast)

    def sat(self):
        return self.clip(0.0, 1.0)

    def maximum(self, c):
        return self.clip(c, np.inf)

    def minimum(self, c):
        return self.clip(-np.inf, c)

    def abs(self):
        return Num(np.abs(self.v), self.e, self.fast)


def stack3(a, b, c):
    return Num(np.stack([a.v, b.v, c.v], -1), np.stack([a.e, b.e, c.e], -1), a.fast)


def dot3(a, b):
    """glam Vec3::dot: x*x' + y*y' + z*z', left to right."""
    return (a.col(0) * b.col(0) + a.col(1) * b.col(1)) + a.col(2) * b.col(2)


def norm3(a):
    """glam normalize: v * (1 / sqrt(dot(v, v)))."""
    return a * (1.0 / dot3(a, a).sqrt()).x3()


def where(mask, a, b):
    m = np.asarray(mask)
    mv = m.reshape(m.shape + (1,) * (a.v.ndim - m.ndim)) if a.v.ndim > m.ndim else m
    return Num(np.where(mv, a.v, b.v), np.where(mv, a.e, b.e), a.fast)


# ---- RNG and seeds (exact) --------------------------------------------------------------------------------------------------

def _pcg(s):
    s = (np.asarray(s, dtype=np.uint64) * 747796405 + 2891336453) & 0xFFFFFFFF
    word = (((s >> ((s >> 28) + 4)) ^ s) * 277803737) & 0xFFFFFFFF
    return s, ((word >> 22) ^ word) & 0xFFFFFFFF


def dispatch_seed(base, frame, k):
    return int(_pcg(np.uint64((base ^ (frame * 64 + k)) & 0xFFFFFFFF))[1])


class WhiteNoise:
    """noise/white.rs: state = seed ^ 48619 x ^ 95461 y (u32); sample() = PCG word as f32 times 2^-32 (the f32 conversion rounds)."""

    def __init__(self, seed, x, y):
        x = np.asarray(x, dtype=np.uint64); y = np.asarray(y, dtype=np.uint64)
        self.s = (np.uint64(seed) ^ ((48619 * x) & 0xFFFFFFFF) ^ ((95461 * y) & 0xFFFFFFFF)) & 0xFFFFFFFF

    def u32(self):
        self.s, w = _pcg(self.s)
        return w

    def sample(self):
        return self.u32().astype(np.float32).astype(np.float64) * 2.0 ** -32


# ---- camera, G-buffer, hit --------------------------------------------------------------------------------------------------

def _hm_mul(a, b):
    f = np.float32
    r = np.zeros(16, np.float32)
    for c in range(4):
        v = b[4 * c:4 * c + 4]
        for k in range(4):
            acc = f(a[k] * v[0]); acc = f(acc + f(a[4 + k] * v[1])); acc = f(acc + f(a[8 + k] * v[2])); acc = f(acc + f(a[12 + k] * v[3]))
            r[4 * c + k] = acc
    return r


def _hm_inverse(m):
    """glam Mat4::inverse (cofactor expansion), evaluated in f32 in glam's order."""
    f = np.float32
    m = [f(x) for x in m]
    m00, m01, m02, m03, m10, m11, m12, m13, m20, m21, m22, m23, m30, m31, m32, m33 = m
    def d(a, b, c, e):
        return f(f(a * b) - f(c * e))
    c00, c02, c03 = d(m22, m33, m32, m23), d(m12, m33, m32, m13), d(m12, m23, m22, m13)
    c04, c06, c07 = d(m21, m33, m31, m23), d(m11, m33, m31, m13), d(m11, m23, m21, m13)
    c08, c10, c11 = d(m21, m32, m31, m22), d(m11, m32, m31, m12), d(m11, m22, m21, m12)
    c12, c14, c15 = d(m20, m33, m30, m23), d(m10, m33, m30, m13), d(m10, m23, m20, m13)
    c16, c18, c19 = d(m20, m32, m30, m22), d(m10, m32, m30, m12), d(m10, m22, m20, m12)
    c20, c22, c23 = d(m20, m31, m30, m21), d(m10, m31, m30, m11), d(m10, m21, m20, m11)
    F0, F1, F2 = [c00, c00, c02, c03], [c04, c04, c06, c07], [c08, c08, c10, c11]
    F3, F4, F5 = [c12, c12, c14, c15], [c16, c16, c18, c19], [c20, c20, c22, c23]
    V0, V1, V2, V3 = [m10, m00, m00, m00], [m11, m01, m01, m01], [m12, m02, m02, m02], [m13, m03, m03, m03]
    sa, sb = [f(1), f(-1), f(1), f(-1)], [f(-1), f(1), f(-1), f(1)]
    r = [f(0)] * 16
    for k in range(4):
        r[k] = f(f(f(f(V1[k] * F0[k]) - f(V2[k] * F1[k])) + f(V3[k] * F2[k])) * sa[k])
        r[4 + k] = f(f(f(f(V0[k] * F0[k]) - f(V2[k] * F3[k])) + f(V3[k] * F4[k])) * sb[k])
        r[8 + k] = f(f(f(f(V0[k] * F1[k]) - f(V1[k] * F3[k])) + f(V3[k] * F5[k])) * sa[k])
        r[12 + k] = f(f(f(f(V0[k] * F2[k]) - f(V1[k] * F4[k])) + f(V2[k] * F5[k])) * sb[k])
    det = f(f(f(f(m[0] * r[0]) + f(m[1] * r[4])) + f(m[2] * r[8])) + f(m[3] * r[12]))
    rcp = f(f(1) / det)
    return np.array([f(x * rcp) for x in r], np.float32)


def ndc_to_world(transform16, projection16):
    """Camera::serialize's ndc_to_world = transform * projection.inverse(), in f32 (exact restatement of the host computation)."""
    t = np.asarray(transform16, np.float32).reshape(16)
    p = np.asarray(projection16, np.float32).reshape(16)
    return _hm_mul(t, _hm_inverse(p))


def camera_ray(n2w, w, h, fast, xs=None, ys=None):
    """Camera::ray for every pixel, or for the pixels (xs, ys): (origin, dir) as Num (H, W, 3) or (N, 3)."""
    m = np.asarray(n2w, np.float64).reshape(4, 4)          # m[c] = column c
    if xs is None:
        ys, xs = np.mgrid[0:h, 0:w].astype(np.float64)
    xs, ys = np.asarray(xs, np.float64), np.asarray(ys, np.float64)
    z = lambda a: Num(a, 0.0, fast)
    nx = (z(xs + 0.5) * 2.0) / float(w) - 1.0
    ny = -((z(ys + 0.5) * 2.0) / float(h) - 1.0)

    def project(zc):
        r = [z(m[0][k]) * nx for k in range(4)]
        r = [r[k] + z(m[1][k]) * ny for k in range(4)]
        r = [r[k] + z(np.full(xs.shape, m[2][k])) * zc for k in range(4)]
        r = [r[k] + m[3][k] for k in range(4)]
        rw = 1.0 / r[3]
        return stack3(r[0] * rw, r[1] * rw, r[2] * rw)

    far, near = project(F32_EPS), project(1.0)
    return near, norm3(far - near)


def oct_decode(e, fast):
    """Normal::decode of exact f32 inputs e (..., 2)."""
    e = np.asarray(e, np.float32).astype(np.float64)
    mx = Num(e[..., 0], 0.0, fast) * 2.0 - 1.0
    my = Num(e[..., 1], 0.0, fast) * 2.0 - 1.0
    nz = (1.0 - mx.abs()) - my.abs()
    t = (-nz).maximum(0.0)
    nx = mx - Num(np.copysign(t.v, mx.v), t.e, fast)
    ny = my - Num(np.copysign(t.v, my.v), t.e, fast)
    return norm3(stack3(nx, ny, nz))


def _bytes(x):
    b = np.asarray(x, np.float32).view(np.uint32).astype(np.int64)
    return [(b >> (8 * k)) & 0xFF for k in range(4)]


def gbuffer(d0, d1, fast):
    """GBufferEntry::unpack (gbuffer.rs:19-57) of the exact G-buffer texels."""
    d0 = np.asarray(d0, np.float32); d1 = np.asarray(d1, np.float32)
    mb, rb, fb, _ = _bytes(d0[..., 3])
    cb = _bytes(d1[..., 3])
    z = lambda a: Num(np.asarray(a, np.float64), 0.0, fast)
    rough = z(rb) / 255.0
    base = np.stack([(cb[k] / 255.0) ** 2.2 for k in range(3)], -1)
    return dict(depth=d0[..., 0].astype(np.float64), normal=oct_decode(d0[..., 1:3], fast), metallic=z(mb) / 255.0,
                roughness=rough * rough, reflectance=z(fb) / 255.0, base=Num(base, base * (POW22_REL + 2.2 * U), fast),
                metallic_byte=mb, some=d0[..., 0] != 0)


def hit(n2w, w, h, d0, d1, fast, xs=None, ys=None):
    """Hit::new(camera.ray(pos), gbuffer): point = origin + dir * (depth - 0.01), for every pixel or for the pixels (xs, ys)."""
    o, d = camera_ray(n2w, w, h, fast, xs, ys)
    if xs is not None:
        d0, d1 = np.asarray(d0, np.float32)[ys, xs], np.asarray(d1, np.float32)[ys, xs]
    g = gbuffer(d0, d1, fast)
    t = Num(g["depth"], 0.0, fast) - _f32c(0.01)
    return dict(g=g, origin=o, dir=d, point=o + d * t.x3())


# ---- BRDFs and lights --------------------------------------------------------------------------------------------------------

def clamped_roughness(g):
    return g["roughness"].clip(CLAMPED_ROUGHNESS_MIN, 1.0)


def specular(g, l, v):
    """SpecularBrdf::eval (brdf.rs:46-79).  Returns (Num (..., 3), undecided mask of the n.l / n.v early-out)."""
    fast = l.fast
    a = clamped_roughness(g)
    n = g["normal"]
    hh = norm3(l + v)
    dl, dv = dot3(n, l), dot3(n, v)
    n_dot_l, n_dot_h, l_dot_h, n_dot_v = dl.sat(), dot3(n, hh).sat(), dot3(l, hh).sat(), dv.sat()
    undecided = (np.abs(dl.v) <= dl.e) | (np.abs(dv.v) <= dv.e)
    zero = (dl.v <= 0) | (dv.v <= 0) | (g["metallic"].v <= 0)
    a2 = a * a
    dd = (n_dot_h * a2 - n_dot_h) * n_dot_h + 1.0
    D = a2 / ((PI * dd) * dd)
    k = a * a / 2.0
    G = (n_dot_v / (n_dot_v * (1.0 - k) + k)) * (n_dot_l / (n_dot_l * (1.0 - k) + k))
    m = g["metallic"]
    r = g["reflectance"]
    f0 = (((_f32c(0.16) * r) * r) * (1.0 - m)).x3() + g["base"] * m.x3()
    c = _f32c(np.float32(50.0) * np.float32(0.33))
    f90 = ((f0.col(0) * c + f0.col(1) * c) + f0.col(2) * c).sat()
    p = (1.0 - l_dot_h).maximum(_f32c(0.001))
    p5 = (p * p) * (p * p) * p
    F = f0 + (f90.x3() - f0) * p5.x3()
    out = (D * G).x3() * F / ((4.0 * n_dot_l) * n_dot_v).x3()
    out = where(zero, Num(np.zeros_like(out.v), 0.0, fast), out)
    return out, undecided & (g["metallic"].v > 0)


def acos_approx(x):
    """glam math::acos_approx (DirectXMath XMScalarACos)."""
    fast = x.fast
    nonneg = x.v >= 0
    ax = x.abs()
    root = (1.0 - ax).maximum(0.0).sqrt()
    cs = [-0.0012624911, 0.0066700901, -0.0170881256, 0.0308918810, -0.0501743046, 0.0889789874, -0.2145988016, 1.5707963050]
    r = Num(np.full(x.v.shape, _f32c(cs[0])), 0.0, fast)
    for c in cs[1:]:
        r = r * ax + _f32c(c)
    r = r * root
    out = where(nonneg, r, PI - r)
    return Num(out.v, out.e + ACOS_BRANCH, fast)


def light_radiance(L, ht, with_spec=True):
    """Light::radiance (light.rs:143-207) for per-pixel light records L (..., 28).  Returns dict(radiance, spec, undecided); with
    with_spec=False only the radiance (what EphemeralSample::pdf reads), without the specular lobe's terms."""
    fast = ht["point"].fast
    L = np.asarray(L, np.float32)
    z = lambda a: Num(np.asarray(a, np.float64), 0.0, fast)
    center, radius, color, rng = z(L[..., 0:3]), z(L[..., 3]), z(L[..., 4:7]), L[..., 7].astype(np.float64)
    kind = L[..., 8].view(np.uint32)
    g, p = ht["g"], ht["point"]
    l = center - p
    sd = oct_decode(L[..., 9:11], fast)
    hv = p - center
    ang = acos_approx(dot3(sd, hv) / (dot3(sd, sd) * dot3(hv, hv)).sqrt())
    q = ang / z(L[..., 11])
    f_angle = where(kind == 1, Num(np.ones(kind.shape), 0.0, fast), (1.0 - (q * q) * q).sat())
    l2 = dot3(l, l)
    inv_r2 = 1.0 / (z(rng) * z(rng))
    factor = l2 * inv_r2
    smooth = (1.0 - factor * factor).sat()
    f_dist = where(np.isinf(rng), Num(np.ones(rng.shape), 0.0, fast), (smooth * smooth) / l2.maximum(_f32c(0.0001)))
    f_cos = dot3(g["normal"], norm3(l)).sat()
    rad = ((color * f_angle.x3()) * f_dist.x3()) * f_cos.x3()
    if not with_spec:
        return dict(radiance=rad)
    v = -ht["dir"]
    n = g["normal"]
    dir_ = ht["dir"]
    r = dir_ - (2.0 * dot3(n, dir_)).x3() * n
    c2r = dot3(l, r).x3() * r - l
    tt = radius * (1.0 / dot3(c2r, c2r).sqrt())
    closest = l + c2r * tt.sat().x3()
    inv_len = 1.0 / dot3(closest, closest).sqrt()
    cr = clamped_roughness(g)
    i_rough = cr / (cr + (radius * 0.5) * inv_len).sat()
    spec, und = specular(g, closest * inv_len.x3(), v)
    spec = (i_rough * i_rough).x3() * spec
    return dict(radiance=rad, spec=spec, undecided=und)


# ---- reservoirs -------------------------------------------------------------------------------------------------------------

def di_fields(res):
    """DiReservoir::read of an (N, 8) buffer: m, w, pdf, occluded, confidence, light point (N, 3), light id."""
    r = np.asarray(res, np.float32).reshape(-1, 8)
    b = r[:, 3].view(np.uint32)
    return dict(m=r[:, 0].astype(np.float64), w=r[:, 1].astype(np.float64), pdf=r[:, 2].astype(np.float64),
                occ=(b & 0xFF) > 0, conf=((b >> 8) & 0xFF).astype(np.float64), point=r[:, 4:7].copy(), id=r[:, 7].view(np.uint32).copy())


def di_resolving(n2w, w, h, d0, d1, lights, res_in, res_out, fast, atm, mutation=None):
    """K10.  `res_in` = the reservoirs it reads (next), `res_out` = what it wrote (prev): the occluded bit there is the visibility the
    kernel traced.  `atm` = atmosphere_inputs(engine): the sky pixels' diffuse output is Atmosphere::sample along the camera ray
    times (1 - 0) / pi (an empty G-buffer entry has metallic 0) and their specular output 0.  Returns dict(diff, spec (Num (H, W,
    3)), conf (H, W), some, undecided, res, sky) where `res` is the (N, 8) reservoir copy expected (with the device's visibility)
    and `sky` the atmosphere restatement of the pixels without a surface (`mutation`: one of SKY_MUTATIONS)."""
    ht = hit(n2w, w, h, d0, d1, fast)
    some = ht["g"]["some"]
    ri, ro = di_fields(res_in), di_fields(res_out)
    occ = ro["occ"].reshape(h, w)
    conf = np.where(ri["occ"].reshape(h, w) == occ, ri["conf"].reshape(h, w), 0.0)
    lights = np.asarray(lights, np.float32).reshape(-1, 28)
    L = lights[np.minimum(ri["id"], len(lights) - 1).reshape(h, w)]
    lr = light_radiance(L, ht)
    rad = lr["radiance"] * Num(ri["w"].reshape(h, w), 0.0, fast).x3()
    zero = Num(np.zeros((h, w, 3)), 0.0, fast)
    rad = where(occ, zero, rad)
    diff = rad * ((1.0 - ht["g"]["metallic"]) / PI).x3()
    spec = rad * where(occ, zero, lr["spec"])
    want = np.asarray(res_in, np.float32).reshape(-1, 8).copy()
    b = want[:, 3].view(np.uint32)
    bits = np.where(some.reshape(-1), (np.where(occ.reshape(-1), 1, 0) | (1 << 8)).astype(np.uint32), b)
    want[:, 3] = bits.view(np.float32)
    sky = atmosphere_sample(atm, ht["dir"][~some], fast, mutation)
    sky["diff"] = sky["lum"] * ((1.0 - Num(np.zeros(len(sky["domain"])), 0.0, fast)) / PI).x3()
    return dict(diff=diff, spec=spec, conf=conf, some=some, undecided=lr["undecided"] & ~occ & some, res=want, sky=sky)


def _mis_m(q0, q1):
    """m(q0, q1) of Mis::eval: 1 where q0 <= 0, else saturate(min(q1 / q0, 1)^8) as three squarings."""
    x = (q1 / q0).minimum(1.0)
    x2 = x * x
    x4 = x2 * x2
    return where(q0.v <= 0, Num(np.ones(q0.v.shape), 0.0, q0.fast), (x4 * x4).sat())


def _ratio(x, y):
    s = x + y
    return where(s.v == 0, Num(np.zeros(s.v.shape), 0.0, x.fast), x / s)


def _decide(r, W, weight):
    """rng * W < weight: (accepted in f64, decided)."""
    p = r * W.v
    margin = weight.v - p
    bound = r * W.e + weight.e + U * np.abs(p) + SUB
    with np.errstate(invalid="ignore"):
        return margin > 0, (~(np.abs(margin) <= bound) | ((margin == 0) & (W.e == 0) & (weight.e == 0))) & np.isfinite(margin)


def _mis_eval(lm, rm, lpdf, lhs_rhs_pdf, rhs_lhs_pdf, rpdf, rhs_jacobian=1.0):
    """Mis::eval (mis.rs:96-145): (m, lhs_mis, rhs_mis).  DI passes rhs_jacobian = 1; the GI spatial merge the texel's jacobian."""
    mm_a, mm_b = _mis_m(rpdf, rhs_lhs_pdf), _mis_m(lhs_rhs_pdf, lpdf)
    mmin = where(mm_a.v <= mm_b.v, mm_a, mm_b)
    mmin = Num(mmin.v, np.maximum(mm_a.e, mm_b.e), lm.fast)
    t = _ratio(lm, rm)
    lhs_mis = t + (1.0 - t) * _ratio(lm * lpdf, rm * lhs_rhs_pdf)
    rhs_mis = (1.0 - t) * _ratio((rm * rpdf) * rhs_jacobian, lm * rhs_lhs_pdf)
    return rm * mmin, lhs_mis, rhs_mis


def half_grid_pairs(w, h, frame, rows=None):
    """The half-width dispatch grid of K7 / K9 (8 * ((ceil(w / 8)) / 2) columns, so with w = 67 the last columns are never reached):
    (gx, gy, lhs x, other x) per pair, resolve_checkerboard_alt / resolve_checkerboard (utils.rs:33-39).  `rows`: only those rows."""
    hw = 8 * (((w + 7) // 8) // 2)
    gy, gx = np.mgrid[0:h, 0:hw]
    gx, gy = gx.reshape(-1), gy.reshape(-1)
    if rows is not None:
        keep = np.isin(gy, rows)
        gx, gy = gx[keep], gy[keep]
    f2 = frame // 2
    return gx, gy, gx * 2 + ((f2 + 1 + gy) % 2), gx * 2 + ((f2 + gy) % 2)


def di_spatial_sample(res_in, stash, seed, frame, w, h, fast, rows=None, flips=0):
    """K9 on every checkerboard pair (or those of `rows`).  `stash`: the (H, W, 4) visibility texels K8 left; or, for the fused
    launch, K7's restatement composed with a visibility per ray (pick_stash), whose pdfs carry bounds and whose undecided pairs are
    skipped.  `flips` is recorded in the candidates (how many visibility bits were flipped to build them).  Returns dict(idx (P,),
    cands: list of dicts of expected (P, 8) words + bound on m / w / pdf, per-pair `allowed` mask per candidate; undecided, skip (P,)
    bool; copies (Q,) indices of the pass-through pixels)."""
    res_in = np.asarray(res_in, np.float32).reshape(-1, 8)
    npx = w * h
    gx, gy, lx, ox = half_grid_pairs(w, h, frame, rows)
    ok = lx < w
    # the other pixel of the pair is copied through only where the lhs is on the screen: the pass returns before the copy otherwise
    # (di_spatial_resampling.rs:230)
    copies = (gy * w + ox)[ok & (ox < w)]
    gx, gy, lx = gx[ok], gy[ok], lx[ok]
    lidx = gy * w + lx
    z = lambda a: Num(np.asarray(a, np.float64), 0.0, fast)
    if isinstance(stash, dict):
        rhs_idx, skip = stash["rhs_idx"][ok], stash["skip"][ok]
        lhs_rhs_vis, rhs_lhs_vis = stash["vis_a"][ok].astype(np.float64), stash["vis_b"][ok].astype(np.float64)
        pdf_lr, pdf_rl = stash["lhs_rhs_pdf"][ok], stash["rhs_lhs_pdf"][ok]
    else:
        stash = np.asarray(stash, np.float32).reshape(h, w, 4)
        ax, bx = gx * 2, gx * 2 + 1
        tz = np.zeros((len(gx), 4), np.float32)
        d0 = np.where((ax < w)[:, None], stash[gy, np.minimum(ax, w - 1)], tz)
        d1 = np.where((bx < w)[:, None], stash[gy, np.minimum(bx, w - 1)], tz)
        rhs_idx, skip = d0[:, 1].view(np.uint32).astype(np.int64), np.zeros(len(gx), bool)
        lhs_rhs_vis, rhs_lhs_vis = d0[:, 0].astype(np.float64), d1[:, 0].astype(np.float64)
        pdf_lr, pdf_rl = z(d1[:, 1]), z(d1[:, 2])
    # K7 writes 0 (no neighbour) or screen index + 1; anything past the frame would make K9 read outside the reservoirs
    assert not ((rhs_idx > 0) & (rhs_idx - 1 >= npx)).any(), "K7 scratch texel holds a neighbour index outside the frame"
    merge = rhs_idx > 0
    lhs = res_in[lidx]
    rhs = res_in[np.where(merge, rhs_idx - 1, 0)]
    lm, lw, lpdf = z(lhs[:, 0]), z(lhs[:, 1]), z(lhs[:, 2])
    rm, rw, rpdf = z(rhs[:, 0]), z(rhs[:, 1]), z(rhs[:, 2])
    # pdf * vis with vis 0 or 1 (K8's texel layout) is exact
    lhs_rhs_pdf = where(lhs_rhs_vis != 0, pdf_lr, z(np.zeros(len(gx))))
    rhs_lhs_pdf = where(rhs_lhs_vis != 0, pdf_rl, z(np.zeros(len(gx))))
    with np.errstate(invalid="ignore", over="ignore"):
        mis_m, lhs_mis, rhs_mis = _mis_eval(lm, rm, lpdf, lhs_rhs_pdf, rhs_lhs_pdf, rpdf)
        wl = (lhs_mis * lpdf) * lw
        wr = (rhs_mis * rhs_lhs_pdf) * rw
        rng = WhiteNoise(seed, lx, gy)
        r1, r2 = rng.sample(), rng.sample()
        W1 = Num(np.zeros(len(gx)), 0.0, fast) + wl
        W2 = W1 + wr
        acc1, dec1 = _decide(r1, W1, wl)
        acc2, dec2 = _decide(r2, W2, wr)
        m_out = lm + mis_m
    cands = []
    for a1 in (False, True):
        for a2 in (False, True):
            allowed = merge & np.where(dec1, acc1 == a1, True) & np.where(dec2, acc2 == a2, True)
            out = np.zeros((len(gx), 8), np.float32)
            src = rhs if a2 else (lhs if a1 else np.zeros_like(lhs))
            pdf = rhs_lhs_pdf if a2 else (lpdf if a1 else z(np.zeros(len(gx))))
            occ = (lhs_rhs_vis == 0) if a2 else ((src[:, 3].view(np.uint32) & 0xFF) > 0)
            conf = (src[:, 3].view(np.uint32) >> 8) & 0xFF
            with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
                wn = W2 / pdf
            # a pdf is either an exact zero or certainly nonzero (K7 decides `pdf > 0` before it builds a ray)
            wv = np.where(pdf.v == 0, 0.0, wn.v)
            we = np.where(pdf.v == 0, 0.0, wn.e)
            out[:, 2] = pdf.v.astype(np.float32)
            out[:, 3] = (occ.astype(np.uint32) | (conf.astype(np.uint32) << 8)).view(np.float32)
            out[:, 4:8] = src[:, 4:8]
            cands.append(dict(allowed=allowed, words=out, m=m_out.v, m_e=m_out.e, w=wv, w_e=we, pdf=pdf.v, pdf_e=pdf.e, flips=flips))
    # no merge: the lhs reservoir goes through as it is
    cands.append(dict(allowed=~merge, words=lhs.copy(), m=lhs[:, 0].astype(np.float64), m_e=np.zeros(len(gx)),
                      w=lhs[:, 1].astype(np.float64), w_e=np.zeros(len(gx)), flips=flips))
    return dict(idx=lidx, cands=cands, undecided=merge & ~(dec1 & dec2) & ~skip, skip=skip, merge=merge, copies=copies)


# ---- K6: temporal resampling -------------------------------------------------------------------------------------------------

LUMA = (_f32c(0.2126), _f32c(0.7152), _f32c(0.0722))
SLOT_KILLED = 0xCAFEBABE


def _take(x, idx):
    """Pixels `idx` (flat) of a per-pixel (H, W, ...) value: Num, array, or a dict of them (a hit)."""
    if isinstance(x, dict):
        return {k: _take(v, idx) for k, v in x.items()}
    if isinstance(x, Num):
        return Num(x.v.reshape((-1,) + x.v.shape[2:])[idx], x.e.reshape((-1,) + x.e.shape[2:])[idx], x.fast)
    a = np.asarray(x)
    return a.reshape((-1,) + a.shape[2:])[idx]


def di_pdf(L, ht, point):
    """DiSample::pdf_ex (di.rs:108-117) with per-pixel light records L (N, 28) and hits ht (N, ...): luma(radiance * (diff + spec))
    of Light::radiance with the base colour set to 1 (Vec3Ext::luma, utils/vec3_ext.rs:52-54; DiffuseBrdf::eval, brdf.rs:20-24), or 0
    for a Light::TYPE_NONE slot or a light point outside the light (Light::contains, light.rs:83-85: |center - point| <= radius).
    Returns (pdf, contains undecided, specular undecided)."""
    fast = ht["point"].fast
    L = np.asarray(L, np.float32)
    g = dict(ht["g"], base=Num(np.ones(ht["g"]["base"].v.shape), 0.0, fast))
    lr = light_radiance(L, dict(ht, g=g))
    diff = (1.0 - g["metallic"]) / PI
    s = lr["radiance"] * (diff.x3() + lr["spec"])
    luma = (s.col(0) * LUMA[0] + s.col(1) * LUMA[1]) + s.col(2) * LUMA[2]
    p = point if isinstance(point, Num) else np.asarray(point, np.float32).astype(np.float64)    # a Num: a bounded light point
    c = Num(L[:, 0:3].astype(np.float64), 0.0, fast) - p
    dist = dot3(c, c).sqrt()
    radius = L[:, 3].astype(np.float64)
    live = L[:, 8].view(np.uint32) != 0
    inside = dist.v <= radius
    pdf = where(live & inside, luma, Num(np.zeros(len(L)), 0.0, fast))
    return pdf, live & (np.abs(radius - dist.v) <= dist.e), live & inside & lr["undecided"]


def _round_u(x):
    """Vec2::round (half away from zero) then as_uvec2 (saturating) of exact f32 inputs."""
    x = np.asarray(x, np.float32).astype(np.float64)
    r = np.where(x < 0, -np.floor(-x + 0.5), np.floor(x + 0.5))
    return np.clip(np.nan_to_num(r, nan=0.0), 0, 2.0 ** 32 - 1).astype(np.int64)


def di_temporal(n2w, n2w_prev, w, h, gb, gb_prev, reproj, lights, res_cur, res_prev, seed, fast, lhs=None, flips=0):
    """K6 di_temporal_resampling::main (di_temporal_resampling.rs:4-112) for every pixel with a surface.  gb / gb_prev: this and the
    previous frame's G-buffer (d0, d1); reproj: the reprojection map (Reprojection::deserialize, reprojection.rs:22-29); res_cur: what
    K5 left in di_reservoirs[1]; res_prev: di_reservoirs[0].  For the fused K5 + K6 launch `lhs` replaces res_cur: K5's sample as
    sampling_lhs restates it, with a bounded w and light point; its skipped pixels are not compared.  `flips` is recorded in the
    candidates (1 where the lhs occluded bit was flipped).
      * lhs: K5's sample, its pdf recomputed with the current light (:47-51).
      * rhs: di_reservoirs[0] at prev_pos().round().as_uvec2() (reprojection.rs:46-48), M clamped to 64 (reservoir.rs:55-57), a killed
        slot zeroes w, a remapped one moves the id to slot - 1 (light.rs:107-129); its hit is rebuilt with the *previous* camera from
        the previous G-buffer (:61-89).
      * Mis::di_temporal (mis.rs:36-65): lhs_rhs_pdf with the rolled-back light (LightsView::get_prev, lights.rs:19-24), rhs_lhs_pdf
        with the current one, 0 for a killed rhs; then Mis::eval, two Reservoir::update and norm_mis (:93-111), confidence 0 for a
        killed rhs and 1 otherwise.
    Every light id dereferenced is asserted to lie inside `lights` (the table as read).  Returns dict(idx, cands, undecided per
    decision type, skip (pixels with an undecided pdf), surf)."""
    f32 = np.float32
    lights = np.asarray(lights, f32).reshape(-1, 28)
    nl = len(lights)
    npx = w * h
    z = lambda a: Num(np.asarray(a, np.float64), 0.0, fast)
    ht = hit(n2w, w, h, gb[0], gb[1], fast)
    idx = np.flatnonzero(ht["g"]["some"].reshape(-1))
    n = len(idx)
    zero = z(np.zeros(n))
    lh = _take(ht, idx)
    prv = di_fields(res_prev)
    if lhs is None:
        cur = di_fields(res_cur)
        lm, lw, lid, lpoint = cur["m"][idx], z(cur["w"][idx]), cur["id"][idx].astype(np.int64), cur["point"][idx]
        locc, lpdf0, lskip = cur["occ"][idx], cur["pdf"][idx], np.zeros(n, bool)
    else:
        assert len(lhs["id"]) == n
        lm, lid, lpoint, locc, lpdf0, lskip = lhs["m"], lhs["id"], lhs["point"], lhs["occ"], lhs["pdf"], lhs["skip"]
        lw = where(locc, z(np.zeros(n)), lhs["w"])      # K5: w is exactly 0 where the shadow ray is occluded
    assert (lid[lm != 0] < nl).all(), "K6 lhs light id outside the light table"
    lid_c = np.minimum(lid, nl - 1)
    lp, und_c1, und_s1 = di_pdf(lights[lid_c], lh, lpoint)
    lpdf = where(lm != 0, lp, z(lpdf0))
    rp = np.asarray(reproj, f32).reshape(-1, 4)[idx]
    has_rp = rp[:, 2] > 0
    rx, ry = _round_u(rp[:, 0]), _round_u(rp[:, 1])
    assert ((rx < w) & (ry < h))[has_rp].all(), "reprojected position outside the frame"
    ridx = ry * w + rx
    read = has_rp & (ridx < npx)
    ri = np.where(read, ridx, 0)
    pick = lambda a, dflt=0: np.where(read.reshape((-1,) + (1,) * (np.ndim(a) - 1)), a[ri], dflt)
    rm = np.minimum(pick(prv["m"]), 64.0)
    rw, rpdf, rocc, rconf, rpoint, rid = pick(prv["w"]), pick(prv["pdf"]), pick(prv["occ"], False), pick(prv["conf"]), pick(prv["point"]), pick(prv["id"]).astype(np.int64)
    ne = rm != 0
    assert (rid[ne] < nl).all(), "K6 rhs light id outside the light table"
    slot = lights[np.minimum(rid, nl - 1), 12].view(np.uint32).astype(np.int64)
    killed = ne & (slot == SLOT_KILLED)
    remap = ne & ~killed & (slot > 0)
    rw = np.where(killed, 0.0, rw)
    rid = np.where(remap, slot - 1, rid)
    assert (rid[remap] < nl).all(), "K6 remapped light id outside the light table"
    rid_c = np.minimum(rid, nl - 1)
    htp = hit(n2w_prev, w, h, gb_prev[0], gb_prev[1], fast)
    rh = _take(htp, ri)
    rhs_some = ne & rh["g"]["some"]
    prev_L = lights[lid_c].copy()
    prev_L[:, 0:12] = lights[lid_c, 16:28]          # Light::rollback (light.rs:137-141)
    lrp, und_c2, und_s2 = di_pdf(prev_L, rh, lpoint)
    use_lr = (lm > 0) & rhs_some
    lhs_rhs_pdf = where(use_lr, lrp, zero)
    rlp, und_c3, und_s3 = di_pdf(lights[rid_c], lh, rpoint)
    use_rl = (rm > 0) & ~killed
    rhs_lhs_pdf = where(use_rl, rlp, zero)
    und = {"contains": (und_c1 & (lm != 0)) | (und_c2 & use_lr) | (und_c3 & use_rl),
           "specular": (und_s1 & (lm != 0)) | (und_s2 & use_lr) | (und_s3 & use_rl)}
    und["K5"] = lskip
    skip = und["contains"] | und["specular"] | lskip
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        lmN, rmN = z(lm), z(rm)
        mis_m, lhs_mis, rhs_mis = _mis_eval(lmN, rmN, lpdf, lhs_rhs_pdf, rhs_lhs_pdf, z(rpdf))
        # m(q0, q1) branches on q0 <= 0: for the recomputed lhs_rhs_pdf that is a decision on a bounded value
        und["mis q0"] = (lhs_rhs_pdf.e > 0) & (lhs_rhs_pdf.v <= lhs_rhs_pdf.e) & (rm > 0)
        m_out = lmN + mis_m
        m_e = np.where(und["mis q0"], np.inf, m_out.e)
        # a recomputed pdf without a finite bound (GGX at minimum roughness on a normal along the view: the (n.h a^2 - n.h) n.h + 1
        # cancellation) leaves the pixel's m and w unbounded: counted
        und["unbounded"] = ~np.isfinite(m_e) | ~np.isfinite(lpdf.e) | ~np.isfinite(lhs_rhs_pdf.e) | ~np.isfinite(rhs_lhs_pdf.e)
        wl = (lhs_mis * lpdf) * lw
        wr = (rhs_mis * rhs_lhs_pdf) * z(rw)
        rng = WhiteNoise(seed, idx % w, idx // w)
        r1, r2 = rng.sample(), rng.sample()
        W1 = zero + wl
        W2 = W1 + wr
        acc1, dec1 = _decide(r1, W1, wl)
        acc2, dec2 = _decide(r2, W2, wr)
    und["update"] = ~(dec1 & dec2)
    conf = np.where(killed, 0, 1).astype(np.uint32)
    cands = []
    for a1 in (False, True):
        for a2 in (False, True):
            allowed = np.where(dec1, acc1 == a1, True) & np.where(dec2, acc2 == a2, True)
            if a2:
                pdf, occ, point, lid_o = rhs_lhs_pdf, rocc, rpoint, rid
            elif a1:
                pdf, occ, point, lid_o = lpdf, locc, lpoint, lid
            else:
                pdf, occ, point, lid_o = zero, np.zeros(n, bool), np.zeros((n, 3), f32), np.zeros(n, np.int64)
            with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
                wn = W2 / pdf
            exact0 = (pdf.v == 0) & (pdf.e == 0)
            firm = pdf.v > pdf.e        # the f32 pdf is certainly nonzero
            out = np.zeros((n, 8), f32)
            out[:, 3] = (occ.astype(np.uint32) | (conf << 8)).view(f32)
            point_e = point.e if isinstance(point, Num) else np.zeros((n, 3))
            out[:, 4:7] = point.v if isinstance(point, Num) else point
            out[:, 7] = lid_o.astype(np.uint32).view(f32)
            cands.append(dict(allowed=allowed, words=out, m=m_out.v, m_e=m_e, pdf=pdf.v, pdf_e=pdf.e,
                              point=point.v if isinstance(point, Num) else out[:, 4:7].astype(np.float64),
                              point_e=point_e, flips=flips,
                              w=np.where(exact0 | ~firm, 0.0, wn.v), w_e=np.where(exact0, 0.0, np.where(firm, wn.e, np.inf))))
    return dict(idx=idx, cands=cands, undecided=und, skip=skip, surf=ht["g"]["some"].reshape(-1), killed=int(killed.sum()),
                remapped=int(remap.sum()), reprojected=int(read.sum()))


def check_temporal(got, res_before, r, what):
    """K6's reservoirs: at every surface pixel without an undecided pdf, one admissible outcome with the discrete words (occluded,
    confidence, light id, and the light point where it is exact) bit for bit and m, w, pdf (and a bounded light point) within their
    bounds; every other pixel untouched.  Returns (largest error / bound ratio, undecided counts per decision type, pixels checked,
    pixels matched only by a candidate with a flipped lhs occluded bit)."""
    got = np.asarray(got, np.float32).reshape(-1, 8)
    before = np.asarray(res_before, np.float32).reshape(-1, 8)
    assert (got[~r["surf"]].view(np.uint32) == before[~r["surf"]].view(np.uint32)).all(), f"{what}: K6 wrote a sky pixel"
    g = got[r["idx"]]
    gb = g.view(np.uint32)
    ok = r["skip"].copy()
    best = np.zeros(len(g))
    found = np.zeros(len(g), bool)
    flips = np.full(len(g), np.inf)
    for c in r["cands"]:
        wb = c["words"].view(np.uint32)
        disc = (gb[:, 3] == wb[:, 3]) & (gb[:, 7] == wb[:, 7])
        rat = []
        with np.errstate(invalid="ignore", divide="ignore"):
            for k, key in ((0, "m"), (1, "w"), (2, "pdf")):
                err = np.abs(g[:, k].astype(np.float64) - c[key])
                rk = np.where(err == 0, 0.0, err / c[key + "_e"])
                rat.append(np.where(np.isnan(rk), np.inf, rk))
            err = np.abs(g[:, 4:7].astype(np.float64) - c["point"])
            rk = np.where(err == 0, 0.0, err / c["point_e"])
            rk = np.where(c["point_e"] == 0, np.where(gb[:, 4:7] == wb[:, 4:7], 0.0, np.inf), np.where(np.isnan(rk), np.inf, rk))
            rat.append(rk.max(1))
        ratio = np.maximum(np.maximum(rat[0], rat[1]), np.maximum(rat[2], rat[3]))
        good = c["allowed"] & disc & (ratio <= 1.0) & ~r["skip"]
        best = np.where(good & ~found, ratio, np.where(good, np.minimum(best, ratio), best))
        flips = np.where(good, np.minimum(flips, c["flips"]), flips)
        found |= good
        ok |= good
    if not ok.all():
        i = np.flatnonzero(~ok)[:4]
        raise AssertionError(f"{what}: {int((~ok).sum())}/{len(ok)} pixels match no admissible outcome; first pixels {r['idx'][i].tolist()}: "
                             f"got {g[i].tolist()}")
    und = {k: int(v.sum()) for k, v in r["undecided"].items()}
    return float(best.max()) if len(best) else 0.0, und, len(g), int((np.isfinite(flips) & (flips > 0)).sum())


def merge_temporal(rs):
    """One K6 restatement whose candidates are those of all of `rs` (the same pixels under different lhs occluded bits)."""
    return dict(rs[0], cands=[c for r in rs for c in r["cands"]], skip=np.logical_or.reduce([r["skip"] for r in rs]),
                undecided={k: np.logical_or.reduce([r["undecided"][k] for r in rs]) for k in rs[0]["undecided"]})


def sampling_lhs(r, sin, cos, trace_any):
    """K5's sample of every surface pixel as k_di_sample_temporal hands it to K6 in registers (di_sampling_px): m 1, pdf 0, the
    light id and w (Num) of the decided selection of `r` (di_sampling), the light point (Num) of Light::ray_bnoise under the decided
    sign of any_orthonormal_pair, and the occluded bit of `trace_any` on the shadow ray rebuilt in strict f32.  Pixels whose selection
    or sign is undecided are marked `skip`."""
    n = len(r["idx"])
    skip = r["undecided"].copy()
    lid, w, we = np.zeros(n, np.int64), np.zeros(n), np.zeros(n)
    for c in r["cands"]:
        sel = c["allowed"] & ~skip      # exactly one candidate where the selection is decided
        lid, w, we = np.where(sel, c["id"], lid), np.where(sel, c["w"], w), np.where(sel, c["w_e"], we)
    L = r["lights"][lid]
    p = r["hit"]["point"]
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        lz = norm3(Num(L[:, 0:3].astype(np.float64), 0.0, p.fast) - p).col(2)
        skip |= ~(np.abs(lz.v) > lz.e)
        point, _ = ray_bnoise(L, p, r["bn"], np.where(lz.v >= 0, 1.0, -1.0))
    pt = hit_point_f32(r["n2w"], r["w"], r["h"], _depth_image(r)).reshape(-1, 3)[r["idx"]]
    occ = np.asarray(trace_any(ray_bnoise_f32(L, pt, r["bn"], sin, cos)), np.uint32) != 0
    return dict(m=np.ones(n), w=Num(w, we, p.fast), pdf=np.zeros(n), occ=occ, point=point, id=lid, skip=skip)


def temporal_tight(r):
    """{key: (tightly bounded, finite nonzero)} for K6's m, w and pdf over the decided outcome of each decided pixel.  m is the
    loosest of the three: Mis::eval raises a ratio of two recomputed pdfs to the 8th power, which multiplies its relative bound by 8."""
    out = {}
    sel0 = ~r["skip"] & ~r["undecided"]["update"] & ~r["undecided"]["unbounded"]
    for key in ("m", "w", "pdf"):
        n = t = 0
        for c in r["cands"]:
            sel = c["allowed"] & sel0
            v, e = c[key][sel], c[key + "_e"][sel]
            fin = np.isfinite(v) & (v != 0)
            n += int(fin.sum()); t += int((e[fin] < 1e-3 * np.abs(v[fin])).sum())
        out[key] = (t, n)
    return out


# fraction of K6's values whose bound must be below 1e-3 relative (temporal_tight).  Cornell with spot lights is the loosest scene
# (H100, strict, 224x126): m 94.1 %, w 98.7 %, pdf 99.4 %; the acos_approx cone term loosens the recomputed pdfs there, and m takes
# their ratio to the 8th power
TIGHT_MIN = {"m": 0.9, "w": 0.98, "pdf": 0.99}


def tight_ok(acc):
    """acc: {key: [tight, n]} summed over frames.  Every key has values and enough of them are tightly bounded."""
    return all(acc[k][1] > 0 and acc[k][0] >= TIGHT_MIN[k] * acc[k][1] for k in TIGHT_MIN)


# ---- K8: visibility of K7's rays -----------------------------------------------------------------------------------------------

def oct_decode_f32(e):
    """Normal::decode (normal.rs) of (..., 2) f32 inputs, evaluated in f32 operation by operation (no contraction), with glam's
    normalize = v * (1 / sqrt(dot(v, v))): the strict build's rounding, exactly."""
    f = np.float32
    e = np.asarray(e, f)
    with np.errstate(invalid="ignore", divide="ignore"):
        mx, my = e[..., 0] * f(2) - f(1), e[..., 1] * f(2) - f(1)
        nz = (f(1) - np.abs(mx)) - np.abs(my)
        t = np.maximum(-nz, f(0))
        nx, ny = mx - np.copysign(t, mx), my - np.copysign(t, my)
        inv = f(1) / np.sqrt((nx * nx + ny * ny) + nz * nz)
        return np.stack([nx * inv, ny * inv, nz * inv], -1).astype(f)


def check_spatial_trace(buf_d0, buf_d1, buf_d2, trace_any, what):
    """K8 di_spatial_resampling::trace (di_spatial_resampling.rs:150-209) on every texel: a texel whose d1 is zero gives d2 = 0; any
    other gives (visibility, d1.z, d1.w, 0) with d1.z / d1.w copied bit for bit, and the visibility is compared with `trace_any` of
    the ray rebuilt from the texels (origin d0.xyz, Normal::decode(d1.xy), length d0.w).  K7's zero ray (origin 0, length 0,
    oct(0) = NaN direction) must come out visible.  Returns (texels traced, visibility disagreements)."""
    d0 = np.asarray(buf_d0, np.float32).reshape(-1, 4)
    d1 = np.asarray(buf_d1, np.float32).reshape(-1, 4)
    d2 = np.asarray(buf_d2, np.float32).reshape(-1, 4)
    b1, b2 = d1.view(np.uint32), d2.view(np.uint32)
    empty = (d1 == 0).all(1)
    assert (b2[empty] == 0).all(), f"{what}: K8 texel with a zero d1 is not zero"
    live = ~empty
    assert (b2[live][:, 1:3] == b1[live][:, 2:4]).all(), f"{what}: K8 d2.yz are not d1.zw"
    assert (b2[live][:, 3] == 0).all() and np.isin(d2[live][:, 0], (0.0, 1.0)).all(), f"{what}: K8 texel layout"
    if not live.any():
        return 0, 0
    rays = np.zeros((int(live.sum()), 8), np.float32)
    rays[:, 0:3] = d0[live][:, 0:3]
    rays[:, 3] = d0[live][:, 3]
    rays[:, 4:7] = oct_decode_f32(d1[live][:, 0:2])
    vis = d2[live][:, 0]
    nan = np.isnan(rays[:, 4:7]).any(1)
    assert (vis[nan] == 1).all(), f"{what}: a ray with an undefined direction (K7's zero ray) is not visible"
    want = 1.0 - np.asarray(trace_any(rays), np.float64)
    return int(live.sum()), int((vis != want).sum())


# ---- K5: DI sampling ---------------------------------------------------------------------------------------------------------

def sincos(a):
    """(sin a, cos a) of a Num angle: 1-Lipschitz, plus the tier's absolute error of the function (SIN_ABS / SIN_ABS_FAST)."""
    k = SIN_ABS_FAST if a.fast else SIN_ABS
    return Num(np.sin(a.v), a.e + k, a.fast), Num(np.cos(a.v), a.e + k, a.fast)


def _ortho_pair(n, sign):
    """glam Vec3::any_orthonormal_pair (Duff et al. 2017) with sign = signum(n.z) given per pixel (+1 / -1)."""
    x, y, z = n.col(0), n.col(1), n.col(2)
    a = -1.0 / (z + sign)
    b = (x * y) * a
    t = stack3(1.0 + (((x * sign) * x) * a), b * sign, -(x * sign))
    bt = stack3(b, ((y * y) * a) + sign, -y)
    return t, bt


def ray_bnoise(L, point, bn, sign):
    """Light::ray_bnoise (light.rs:217-239) for light records L (N, 28), hit points `point` (Num (N, 3)) and blue-noise texels bn
    (N, 4 bytes; BlueNoise::first_sample = bytes x, y over 255).  Returns (light point = hit + dir * distance, distance)."""
    fast = point.fast
    z = lambda a: Num(np.asarray(a, np.float64), 0.0, fast)
    to_light = z(L[:, 0:3]) - point
    light_dir = norm3(to_light)
    dist = dot3(to_light, to_light).sqrt()
    light_radius = z(L[:, 3]) / dist
    tg, bt = _ortho_pair(light_dir, sign)
    angle = (z(bn[:, 0]) / 255.0) * _f32c(np.float32(2.0) * np.float32(np.pi))
    radius = (z(bn[:, 1]) / 255.0).sqrt()
    sa, ca = sincos(angle)
    dx, dy = (sa * radius) * light_radius, (ca * radius) * light_radius
    rd = norm3((light_dir + dx.x3() * tg) + dy.x3() * bt)
    return point + rd * dist.x3(), dist


def hit_point_f32(n2w, w, h, depth):
    """Hit::new's point for every pixel, evaluated in f32 operation by operation as the strict build does: Camera::ray (camera.rs:80-93,
    glam project_point3 and normalize) and origin + dir * (depth - 0.01)."""
    f = np.float32
    m = np.asarray(n2w, f).reshape(4, 4)
    ys, xs = np.mgrid[0:h, 0:w].astype(f)
    nx = (((xs + f(0.5)) * f(2)) / f(w)) - f(1)
    ny = -((((ys + f(0.5)) * f(2)) / f(h)) - f(1))

    def project(zc):
        r = [m[0][k] * nx for k in range(4)]
        r = [r[k] + m[1][k] * ny for k in range(4)]
        r = [r[k] + m[2][k] * zc for k in range(4)]
        r = [r[k] + m[3][k] for k in range(4)]
        rw = f(1) / r[3]
        return np.stack([r[0] * rw, r[1] * rw, r[2] * rw], -1)

    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        far, near = project(f(F32_EPS)), project(f(1))
        d = far - near
        d = d * (f(1) / np.sqrt((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]))[..., None]
        t = np.asarray(depth, f) - f(0.01)
        return (near + d * t[..., None]).astype(f)


def ray_bnoise_f32(L, point, bn, sin, cos):
    """Light::ray_bnoise in f32 operation by operation (the strict build's rounding, with its sin / cos passed in): (N, 8) rays
    (origin = light point, length, direction = -dir) for `trace_any`."""
    f = np.float32
    L = np.asarray(L, f)
    p = np.asarray(point, f)
    d3 = lambda a, b: (a[:, 0] * b[:, 0] + a[:, 1] * b[:, 1]) + a[:, 2] * b[:, 2]
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        tl = L[:, 0:3] - p
        ld = tl * (f(1) / np.sqrt(d3(tl, tl)))[:, None]
        dist = np.sqrt(d3(tl, tl))
        lr = L[:, 3] / dist
        x, y, zz = ld[:, 0], ld[:, 1], ld[:, 2]
        s = np.copysign(f(1), zz).astype(f)
        a = f(-1) / (s + zz)
        b = (x * y) * a
        tg = np.stack([f(1) + ((s * x) * x) * a, s * b, -(s * x)], -1)
        bt = np.stack([b, s + (y * y) * a, -y], -1)
        ang = (bn[:, 0].astype(f) / f(255)) * f(f(2) * f(np.pi))
        rad = np.sqrt(bn[:, 1].astype(f) / f(255))
        sa, ca = np.asarray(sin(ang), f), np.asarray(cos(ang), f)
        dx, dy = (sa * rad) * lr, (ca * rad) * lr
        rd = (ld + dx[:, None] * tg) + dy[:, None] * bt
        rd = rd * (f(1) / np.sqrt(d3(rd, rd)))[:, None]
        rays = np.zeros((len(L), 8), f)
        rays[:, 0:3] = p + rd * dist[:, None]
        rays[:, 3] = dist
        rays[:, 4:7] = -rd
    return rays


def di_sampling(n2w, w, h, d0, d1, lights, light_count, blue_noise, seed, frame, fast):
    """K5 di_sampling::main (di_sampling.rs:4-94) with EphemeralReservoir::build (ephemeral.rs:14-55) for every pixel with a surface:
    max_samples = min(light_count, 16) candidates, light id = sample_int() % light_count (exact), candidate pdf = sqrt(luma(radiance))
    (EphemeralSample::pdf, utils/vec3_ext.rs:56-58: the radiance alone, no BRDF), weight = pdf * f32(light_count), Reservoir::update
    and norm_avg (reservoir.rs:24-39, :63-79).  The running sum W does not depend on which candidates were taken, so the consistent
    final selections are the last decided accept plus every undecided step after it (and no selection at all when nothing was decided
    accepted: light 0 with w = 0).  Returns dict(idx, surf, cands (id, w, w_e, allowed), undecided update, hit, bn, lights, ms).
    light_count = 0 (the reference's zero reservoir) is not restated: the engine's sun always holds slot 0, so no frame has it."""
    lights = np.asarray(lights, np.float32).reshape(-1, 28)
    nl, lc = len(lights), int(light_count)
    assert lc > 0, "K5 restatement: light_count = 0 (the sun always holds slot 0)"
    ht = hit(n2w, w, h, d0, d1, fast)
    surf = ht["g"]["some"].reshape(-1)
    idx = np.flatnonzero(surf)
    n = len(idx)
    lh = _take(ht, idx)
    xs, ys = idx % w, idx // w
    bn = np.asarray(blue_noise, np.uint8).reshape(256, 256, 4)[(ys + 11 * frame) % 256, (xs + 71 * frame) % 256]   # blue.rs:15-19
    ms = min(lc, 16)
    rng = WhiteNoise(seed, xs, ys)
    W = Num(np.zeros(n), 0.0, fast)
    steps = []
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        for _ in range(ms):
            lid = (rng.u32() % lc).astype(np.int64)
            assert (lid < nl).all(), "K5 light id outside the light table"
            rad = light_radiance(lights[lid], lh, with_spec=False)["radiance"]
            pdf = ((rad.col(0) * LUMA[0] + rad.col(1) * LUMA[1]) + rad.col(2) * LUMA[2]).sqrt()
            weight = pdf * float(np.float32(lc))
            W = W + weight
            acc, dec = _decide(rng.sample(), W, weight)
            steps.append((lid, pdf, acc, dec))
        last = np.full(n, -1)
        for k, (_, _, acc, dec) in enumerate(steps):
            last = np.where(dec & acc, k, last)
        cands = [dict(id=np.zeros(n, np.int64), w=np.zeros(n), w_e=np.zeros(n), allowed=last < 0)]
        for k, (lid, pdf, acc, dec) in enumerate(steps):
            wn = W / (pdf * float(ms))
            exact0 = (pdf.v == 0) & (pdf.e == 0)
            firm = pdf.v > pdf.e        # the f32 pdf, and so the denominator, is certainly nonzero
            cands.append(dict(id=lid, w=np.where(exact0 | ~firm, 0.0, wn.v), w_e=np.where(exact0, 0.0, np.where(firm, wn.e, np.inf)),
                              allowed=(last == k) | (~dec & (k > last))))
    und = np.zeros(n, bool)
    for _, _, _, dec in steps:
        und |= ~dec
    return dict(idx=idx, surf=surf, cands=cands, undecided=und, hit=lh, bn=bn, lights=lights, ms=ms, w=w, h=h, n2w=n2w,
                depth=np.asarray(d0, np.float32).reshape(-1, 4)[idx, 0])


def check_sampling(got, res_before, r, sin, cos, trace_any, what):
    """K5's reservoirs against the restatement.  Sky pixels are left as they were; at every surface pixel m = 1 exactly, pdf 0, bytes (occluded, confidence 0), the light id one of a consistent selection's, w within
    that selection's bound (exactly 0 when occluded) and the light point (the shadow ray's origin) within its bound, under either sign
    of any_orthonormal_pair where signum(light_dir.z) is undecided.  The occluded bit is compared with `trace_any` of the shadow ray
    rebuilt in strict f32 (ray_bnoise_f32 on hit_point_f32); the rebuilt light point is returned for a bit-exact comparison in the
    strict tier.  Returns dict(ratio (largest w / light point error over its bound), undecided (selection, sign), n, traced, disagree,
    tight w / light point [tightly bounded, finite nonzero], lp_f32 (the rebuilt light points), got (the checked words))."""
    got = np.asarray(got, np.float32).reshape(-1, 8)
    before = np.asarray(res_before, np.float32).reshape(-1, 8)
    surf = r["surf"]
    assert (got[~surf].view(np.uint32) == before[~surf].view(np.uint32)).all(), f"{what}: K5 wrote a sky pixel"
    g = got[r["idx"]]
    gb = g.view(np.uint32)
    out = dict(ratio=0.0, undecided={"update": int(r["undecided"].sum()), "sign": 0}, n=len(g), traced=0, disagree=0,
               tight={"w": [0, 0], "light_point": [0, 0]}, lp_f32=np.zeros((len(g), 3), np.float32), got=g)
    assert (g[:, 0] == 1).all() and (gb[:, 2] == 0).all(), f"{what}: K5's m must be 1 and its pdf 0"
    occ = gb[:, 3]
    assert np.isin(occ, (0, 1)).all(), f"{what}: K5's bytes must be (occluded, confidence 0)"
    occ = occ == 1
    assert (gb[occ, 1] == 0).all(), f"{what}: K5's w must be exactly 0 where the shadow ray is occluded"
    gid = gb[:, 7].astype(np.int64)
    ok = np.zeros(len(g), bool)
    best = np.full(len(g), np.inf)
    for c in r["cands"]:
        with np.errstate(invalid="ignore", divide="ignore"):
            err = np.abs(g[:, 1].astype(np.float64) - c["w"])
            rk = np.where(err == 0, 0.0, err / c["w_e"])
        rk = np.where(occ, 0.0, np.where(np.isnan(rk), np.inf, rk))
        good = c["allowed"] & (gid == c["id"]) & (rk <= 1.0)
        best = np.where(good, np.minimum(best, rk), best)
        ok |= good
        dec = c["allowed"] & ~r["undecided"]
        fin = dec & ~occ & np.isfinite(c["w"]) & (c["w"] != 0)
        out["tight"]["w"][0] += int((c["w_e"][fin] < 1e-3 * np.abs(c["w"][fin])).sum()); out["tight"]["w"][1] += int(fin.sum())
    if not ok.all():
        i = np.flatnonzero(~ok)[:4]
        raise AssertionError(f"{what}: {int((~ok).sum())}/{len(ok)} K5 pixels match no consistent selection; first pixels "
                             f"{r['idx'][i].tolist()}: got {g[i].tolist()}")
    assert (gid < len(r["lights"])).all()
    L = r["lights"][gid]
    p = r["hit"]["point"]
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        lz = norm3(Num(L[:, 0:3].astype(np.float64), 0.0, p.fast) - p).col(2)     # light_dir.z, whose signum ortho_pair takes
        # glam's signum(-0.0) is -1 (as the rebuild's copysign is): a z that may be +-0 in f32, an exact 0 included, is undecided
        sign_und = ~(np.abs(lz.v) > lz.e)
        out["undecided"]["sign"] = int(sign_und.sum())
        pos = np.where(lz.v >= 0, 1.0, -1.0)
        lp_ok = np.zeros(len(g), bool)
        lp_best = np.full(len(g), np.inf)
        for s in (1.0, -1.0):
            allowed = sign_und | (pos == s)
            lp, _ = ray_bnoise(L, p, r["bn"], np.full(len(g), s))
            err = np.abs(g[:, 4:7].astype(np.float64) - lp.v)
            rk = np.where(err == 0, 0.0, err / lp.e)
            rk = np.where(np.isnan(rk), np.inf, rk).max(1)
            good = allowed & (rk <= 1.0)
            lp_best = np.where(good, np.minimum(lp_best, rk), lp_best)
            lp_ok |= good
            # a coordinate's bound relative to the point's largest coordinate: a coordinate near 0 carries the rounding of the others
            sel = allowed & ~sign_und
            v, e = lp.v[sel], lp.e[sel]
            scale = np.abs(v).max(1, keepdims=True) + 0 * v
            fin = np.isfinite(scale) & (scale != 0)
            out["tight"]["light_point"][0] += int((e[fin] < 1e-3 * scale[fin]).sum()); out["tight"]["light_point"][1] += int(fin.sum())
    if not lp_ok.all():
        i = np.flatnonzero(~lp_ok)[:4]
        raise AssertionError(f"{what}: {int((~lp_ok).sum())}/{len(g)} K5 light points outside their bound; first pixels "
                             f"{r['idx'][i].tolist()}: got {g[i, 4:7].tolist()}")
    out["ratio"] = float(max(best.max(), lp_best.max())) if len(g) else 0.0
    pt = hit_point_f32(r["n2w"], r["w"], r["h"], _depth_image(r)).reshape(-1, 3)[r["idx"]]
    rays = ray_bnoise_f32(L, pt, r["bn"], sin, cos)
    out["lp_f32"] = rays[:, 0:3].copy()
    want = np.asarray(trace_any(rays), np.uint32) != 0
    out["traced"], out["disagree"] = len(g), int((want != occ).sum())
    return out


# fraction of K5's w and light points whose bound must be below 1e-3 relative (check_sampling's "tight" counts; a light point
# coordinate against the point's largest coordinate).  Loosest w measured on an H100: 96.7 % (edge test, Cornell with 16 lights, fast
# build), 97.2 % (Cornell with spot lights, 224x126, fast build); 98.1 % on the strict oracle (spot lights, 72x48).  Near a cone's edge
# the candidate pdf sqrt(luma) is small and carries the acos_approx slack.  Every light point measured was tightly bounded.
SAMPLING_TIGHT_MIN = {"w": 0.95, "light_point": 0.99}


def sampling_tight_ok(acc):
    return all(acc[k][1] > 0 and acc[k][0] >= SAMPLING_TIGHT_MIN[k] * acc[k][1] for k in SAMPLING_TIGHT_MIN)


def _depth_image(r):
    d = np.zeros(r["w"] * r["h"], np.float32)
    d[r["idx"]] = r["depth"]
    return d.reshape(r["h"], r["w"])


# ---- K7: DI spatial tap choice -------------------------------------------------------------------------------------------------

K7_BRANCHES = ("self tap", "sky or outside", "depth", "normal", "radius floor", "exhausted", "empty neighbour")
K7_UNDECIDED = ("truncation", "depth", "normal", "pdf", "fold")


def _trunc_decided(x):
    """as_ivec2 truncates toward zero: decided where trunc is the same over [v - e, v + e] (its steps are at the nonzero integers)."""
    with np.errstate(invalid="ignore"):
        return np.trunc(x.v - x.e) == np.trunc(x.v + x.e)


def _contain(x, w):
    """Camera::contain (camera.rs:57-77) on one coordinate: mirror below 0, then above the screen.  On screens smaller than the tap
    radius the result can be negative; cast to u32 it lies outside the frame."""
    x = np.where(x < 0, -x, x)
    return np.where(x >= w, w - x + w - 1, x)


def oct_encode(n):
    """Normal::encode (normal.rs:9-23) of a Num direction (N, 3): (encoded Num (N, 2), decided).  The fold (n.z >= 0) and, below
    the equator, the copysign of x and y are decisions, decided where the value is farther from 0 than its bound."""
    s = (n.col(0).abs() + n.col(1).abs()) + n.col(2).abs()
    q = n / s.x3()
    x, y, zc = q.col(0), q.col(1), q.col(2)
    up = zc.v >= 0
    dec = np.abs(zc.v) > zc.e
    dec &= up | ((np.abs(x.v) > x.e) & (np.abs(y.v) > y.e))
    tx, ty = 1.0 - y.abs(), 1.0 - x.abs()
    ex = where(up, x, Num(np.copysign(tx.v, x.v), tx.e, n.fast)) * 0.5 + 0.5
    ey = where(up, y, Num(np.copysign(ty.v, y.v), ty.e, n.fast)) * 0.5 + 0.5
    return Num(np.stack([ex.v, ey.v], -1), np.stack([ex.e, ey.e], -1), n.fast), dec


def di_spatial_pick(n2w, w, h, d0, d1, lights, res, seed, frame, fast, rows=None):
    """K7 di_spatial_resampling::pick (di_spatial_resampling.rs:4-147) on every pair of the half-width grid (or those of `rows`).
      * lhs = resolve_checkerboard_alt(id, frame / 2) (utils.rs:37-39); off the screen: nothing is written (state 0); a sky lhs: the
        two d1 texels are cleared (state 1; the reference leaves them stale, C-15).
      * 8 tries: WhiteNoise::sample_disk (noise/white.rs:44-56: radius = sqrt(sample) first, then the angle sample * PI * 2, (cos, sin)
        * radius) times max_radius, plus the lhs position; as_ivec2 truncates toward zero before Camera::contain mirrors.  A tap on the
        lhs itself uses up its try.  A tap outside the frame reads zero and, like the sky, a depth off by more than 0.33 of the lhs
        depth or a normal dot below 0.33 (both from GBufferEntry::unpack of the neighbour's texels), is rejected and halves
        max_radius with a floor of 5; an accepted neighbour with an empty reservoir (M = 0) does not halve it.
      * found: lhs_rhs_pdf = lhs.pdf(rhs_hit), rhs_lhs_pdf = rhs.pdf(lhs_hit) (DiSample::pdf, di.rs:95-117); a ray where the pdf is
        > 0 (DiSample::ray, di.rs:119-123: origin the light point, dir = normalize(hit - light point), len = |hit - light point|),
        else the zero ray (origin 0, len 0, Normal::encode(0) = NaN).  Texel a = (ray_a origin, len), (encode(dir_a), rhs_idx + 1, 0);
        texel b = (ray_b origin, len), (encode(dir_b), lhs_rhs_pdf, rhs_lhs_pdf) (state 2); no neighbour: d1 texels cleared (state 1).
    Every decision (truncation, the depth and normal tests, pdf > 0, the fold signs) is decided only where its margin exceeds its
    bound; a pair with an undecided one is counted and skipped.  Returns dict(pairs (gx, gy, lx), state (P,), undecided (P,),
    und (counts per decision), branches (counts per K7_BRANCHES), and for the found pairs: found (P,) mask and per-found-pair rhs_idx,
    lhs / rhs light point, len_a / len_b / enc_a / enc_b (Num), zero_a / zero_b, lhs_rhs_pdf / rhs_lhs_pdf (Num))."""
    d0 = np.asarray(d0, np.float32).reshape(h, w, 4)
    d1 = np.asarray(d1, np.float32).reshape(h, w, 4)
    lights = np.asarray(lights, np.float32).reshape(-1, 28)
    nl = len(lights)
    rf = di_fields(res)
    gx, gy, lx, _ = half_grid_pairs(w, h, frame, rows)
    npair = len(gx)
    state = np.zeros(npair, np.int64)
    on = lx < w
    depth = d0[..., 0]
    surf = on & (depth[gy, np.minimum(lx, w - 1)] != 0)
    state[on] = 1
    und = np.zeros(npair, bool)
    und_n = dict.fromkeys(K7_UNDECIDED, 0)
    br = dict.fromkeys(K7_BRANCHES, 0)
    P = np.flatnonzero(surf)
    n = len(P)
    px, py = lx[P], gy[P]
    z = lambda a: Num(np.asarray(a, np.float64), 0.0, fast)
    dl = z(depth[py, px])
    nrm_l = oct_decode(d0[py, px, 1:3], fast)
    rng = WhiteNoise(seed, px, py)
    radius = np.full(n, 128.0)
    active = np.ones(n, bool)
    u = np.zeros(n, bool)
    found = np.zeros(n, bool)
    floor = np.zeros(n, bool)
    rx, ry = np.zeros(n, np.int64), np.zeros(n, np.int64)
    thr = _f32c(0.33)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        for _ in range(8):
            r = z(rng.sample()).sqrt()
            ang = (z(rng.sample()) * PI) * 2.0
            sa, ca = sincos(ang)
            fx = (ca * r) * radius + px.astype(np.float64)
            fy = (sa * r) * radius + py.astype(np.float64)
            dec = _trunc_decided(fx) & _trunc_decided(fy)
            und_n["truncation"] += int((active & ~dec).sum())
            u |= active & ~dec
            active &= dec
            tx = _contain(np.trunc(fx.v).astype(np.int64), w)
            ty = _contain(np.trunc(fy.v).astype(np.int64), h)
            self_ = active & (tx == px) & (ty == py)
            br["self tap"] += int(self_.sum())
            live = active & ~self_
            inside = (tx >= 0) & (ty >= 0) & (tx < w) & (ty < h)
            cx, cy = np.clip(tx, 0, w - 1), np.clip(ty, 0, h - 1)
            dr = np.where(inside, depth[cy, cx], 0.0)
            rej_sky = live & (dr == 0)
            live &= ~rej_sky
            diff = (z(dr) - dl).abs()
            lim = dl * thr
            margin, bound = diff.v - lim.v, diff.e + lim.e
            dec = (np.abs(margin) > bound) | (bound == 0)
            und_n["depth"] += int((live & ~dec).sum())
            u |= live & ~dec
            live &= dec
            rej_depth = live & (margin > 0)
            live &= ~rej_depth
            dt = dot3(oct_decode(d0[cy, cx, 1:3], fast), nrm_l)
            margin, bound = dt.v - thr, dt.e
            dec = (np.abs(margin) > bound) | (bound == 0)
            und_n["normal"] += int((live & ~dec).sum())
            u |= live & ~dec
            live &= dec
            rej_normal = live & (margin < 0)
            live &= ~rej_normal
            br["sky or outside"] += int(rej_sky.sum()); br["depth"] += int(rej_depth.sum()); br["normal"] += int(rej_normal.sum())
            rej = rej_sky | rej_depth | rej_normal
            radius = np.where(rej, np.maximum(radius * 0.5, 5.0), radius)
            floor |= rej & (radius == 5.0)
            nonempty = rf["m"][np.where(live, cy * w + cx, 0)] != 0
            br["empty neighbour"] += int((live & ~nonempty).sum())
            hitn = live & nonempty
            rx, ry = np.where(hitn, cx, rx), np.where(hitn, cy, ry)
            found |= hitn
            active &= ~u & ~hitn
    br["radius floor"] = int((floor & ~u).sum())
    br["exhausted"] = int((~found & ~u).sum())
    F = np.flatnonzero(found)
    lidx, ridx = py[F] * w + px[F], ry[F] * w + rx[F]
    lid, rid = rf["id"][lidx].astype(np.int64), rf["id"][ridx].astype(np.int64)
    assert (lid < nl).all() and (rid < nl).all(), "K7 light id outside the light table"
    lp, rp = rf["point"][lidx], rf["point"][ridx]
    lh = hit(n2w, w, h, d0, d1, fast, px[F], py[F])
    rh = hit(n2w, w, h, d0, d1, fast, rx[F], ry[F])
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        pdf_lr, uc1, us1 = di_pdf(lights[lid], rh, lp)
        pdf_rl, uc2, us2 = di_pdf(lights[rid], lh, rp)
        pos_lr, pos_rl = pdf_lr.v > pdf_lr.e, pdf_rl.v > pdf_rl.e
        zero_lr, zero_rl = (pdf_lr.v == 0) & (pdf_lr.e == 0), (pdf_rl.v == 0) & (pdf_rl.e == 0)
        upd = uc1 | us1 | uc2 | us2 | ~(pos_lr | zero_lr) | ~(pos_rl | zero_rl)

        def ray(point, ht):
            d = ht["point"] - z(point)
            ln = dot3(d, d).sqrt()
            enc, dec = oct_encode(d * (1.0 / ln).x3())
            return ln, enc, dec
        len_a, enc_a, dec_a = ray(lp, rh)
        len_b, enc_b, dec_b = ray(rp, lh)
    ufold = ~upd & ((pos_lr & ~dec_a) | (pos_rl & ~dec_b))
    und_n["pdf"] = int(upd.sum()); und_n["fold"] = int(ufold.sum())
    u[F] |= upd | ufold
    und[P] = u
    st = np.where(found, 2, 1)
    state[P] = st
    return dict(pairs=(gx, gy, lx), state=state, undecided=und, und=und_n, branches=br, found=P[F], rhs_idx=ridx + 1,
                lhs_point=lp, rhs_point=rp, len_a=len_a, len_b=len_b, enc_a=enc_a, enc_b=enc_b, zero_a=~pos_lr, zero_b=~pos_rl,
                lhs_rhs_pdf=pdf_lr, rhs_lhs_pdf=pdf_rl, found_und=u[F], w=w, h=h, n2w=n2w, depth=depth)


def check_spatial_pick(got_d0, got_d1, before_d0, before_d1, r, what):
    """K7's scratch texels against the restatement, at every pair that is not undecided: state 0 pairs and the columns past the
    grid untouched; state 1: both d1 texels zero, d0 as it was; state 2: rhs_idx + 1 exact, ray origins the light points' words
    exactly (zero for a zero ray), lengths, encoded directions and pdfs within their bounds (a zero ray: length 0, NaN direction).
    Texel b at x = w is dropped.  Returns dict(ratio, undecided, pairs, tight [bounded below 1e-3 relative, finite nonzero])."""
    w, h = r["w"], r["h"]
    gd0, gd1 = (np.asarray(a, np.float32).reshape(h * w, 4) for a in (got_d0, got_d1))
    bd0, bd1 = (np.asarray(a, np.float32).reshape(h * w, 4) for a in (before_d0, before_d1))
    gx, gy, lx = r["pairs"]
    ax, bx = gx * 2, gx * 2 + 1
    ia, ib = gy * w + ax, gy * w + np.minimum(bx, w - 1)
    bin_ = bx < w
    # the texels of the checked rows that no decided pair may write: both buffers as they were
    keep = np.isin(np.arange(h * w) // w, gy)
    und = r["undecided"]
    skip = np.zeros(h * w, bool)
    skip[ia[und]] = True; skip[ib[und & bin_]] = True
    s0 = r["state"] == 0
    for b, g, nm in ((bd0, gd0, "d0"), (bd1, gd1, "d1")):
        untouched = keep & ~skip
        for st in (1, 2):
            sel = (r["state"] == st) & ~und
            if st == 2 or nm == "d1":
                untouched[ia[sel]] = False; untouched[ib[sel & bin_]] = False
        assert (g[untouched].view(np.uint32) == b[untouched].view(np.uint32)).all(), f"{what}: K7 wrote a texel it should leave ({nm})"
    s1 = (r["state"] == 1) & ~und
    for i in (ia[s1], ib[s1 & bin_]):
        assert (gd1[i].view(np.uint32) == 0).all(), f"{what}: K7 state-1 d1 texel is not zero"
    assert not s0[und].any()
    F = r["found"]
    fu = r["found_und"]
    F, sel = F[~fu], ~fu
    a, b, inb = ia[F], ib[F], bin_[F]
    out = dict(ratio=0.0, undecided=int(und.sum()), pairs=int((~s0).sum()), tight=[0, 0])
    ba1, bb1 = gd1[a].view(np.uint32), gd1[b].view(np.uint32)
    assert (ba1[:, 2] == r["rhs_idx"][sel].astype(np.uint32)).all(), f"{what}: K7 rhs_idx + 1"
    assert (ba1[:, 3] == 0).all(), f"{what}: K7 texel a d1.w"
    worst = [0.0]

    def within(got, num, key, mask):
        v, e = num.v[sel][mask], num.e[sel][mask]
        gg = got[mask].astype(np.float64)
        err = np.abs(gg - v)
        with np.errstate(invalid="ignore", divide="ignore"):
            rk = np.where(err == 0, 0.0, err / e)
        rk = np.where(np.isnan(rk), np.inf, rk)
        if not (rk <= 1).all():
            i = np.flatnonzero(~(rk <= 1).reshape(len(rk), -1).all(1))[:4]
            raise AssertionError(f"{what}: K7 {key} outside its bound at pairs {F[mask][i].tolist()}: got {gg[i].tolist()} want "
                                 f"{v[i].tolist()} bound {e[i].tolist()}")
        worst[0] = max(worst[0], float(rk.max()) if rk.size else 0.0)
        if key in ("len", "pdf"):
            fin = np.isfinite(v) & (v != 0)
            out["tight"][0] += int((e[fin] < 1e-3 * np.abs(v[fin])).sum()); out["tight"][1] += int(fin.sum())

    for tex0, tex1, key, mask in ((gd0[a], gd1[a], "a", np.ones(len(F), bool)), (gd0[b], gd1[b], "b", inb)):
        zr = r["zero_" + key][sel]
        pt = r["lhs_point" if key == "a" else "rhs_point"][sel]
        live = mask & ~zr
        assert (tex0[live][:, 0:3].view(np.uint32) == pt[live].view(np.uint32)).all(), f"{what}: K7 ray {key} origin"
        dead = mask & zr
        assert (tex0[dead].view(np.uint32) == 0).all() and np.isnan(tex1[dead][:, 0:2]).all(), f"{what}: K7 zero ray {key}"
        within(tex0[:, 3], r["len_" + key], "len", live)
        within(tex1[:, 0:2], r["enc_" + key], "direction", live)
    within(gd1[b][:, 2], r["lhs_rhs_pdf"], "pdf", inb)
    within(gd1[b][:, 3], r["rhs_lhs_pdf"], "pdf", inb)
    out["ratio"] = worst[0]
    return out


def di_ray_f32(point, hit_pt):
    """DiSample::ray evaluated in f32 operation by operation, with the direction through the octahedral round trip (Normal::encode,
    then Normal::decode as the trace pass does): the strict build's (N, 8) ray, exactly."""
    f = np.float32
    p, q = np.asarray(point, f), np.asarray(hit_pt, f)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        d = q - p
        ln = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
        n = d * (f(1) / ln)[:, None]
        n = n / ((np.abs(n[:, 0]) + np.abs(n[:, 1])) + np.abs(n[:, 2]))[:, None]
        up = n[:, 2] >= 0
        ex = np.where(up, n[:, 0], np.copysign(f(1) - np.abs(n[:, 1]), n[:, 0]))
        ey = np.where(up, n[:, 1], np.copysign(f(1) - np.abs(n[:, 0]), n[:, 1]))
        enc = np.stack([ex * f(0.5) + f(0.5), ey * f(0.5) + f(0.5)], -1).astype(f)
    rays = np.zeros((len(p), 8), f)
    rays[:, 0:3], rays[:, 3], rays[:, 4:7] = p, ln, oct_decode_f32(enc)
    return rays


def pick_stash(r, trace_any):
    """K9's per-pair inputs as the fused launch makes them from K7's pairs: rhs_idx (0 without a neighbour), the two pdfs (Num; 0 at
    texel b's x = w, which the launch does not trace) and the visibility of each ray from `trace_any` of the ray rebuilt in strict f32
    (a zero ray is visible).  Returns the dict di_spatial_sample takes, plus `rays_b` (the pairs whose texel b is traced)."""
    gx, gy, lx = r["pairs"]
    w = r["w"]
    npair = len(gx)
    fast = r["len_a"].fast
    rhs_idx = np.zeros(npair, np.int64)
    vis_a, vis_b = np.zeros(npair), np.zeros(npair)
    zero = Num(np.zeros(npair), 0.0, fast)
    plr, prl = Num(zero.v.copy(), zero.e.copy(), fast), Num(zero.v.copy(), zero.e.copy(), fast)
    F = r["found"]
    inb = (gx[F] * 2 + 1) < w
    rhs_idx[F] = r["rhs_idx"]
    plr.v[F] = np.where(inb, r["lhs_rhs_pdf"].v, 0.0); plr.e[F] = np.where(inb, r["lhs_rhs_pdf"].e, 0.0)
    prl.v[F] = np.where(inb, r["rhs_lhs_pdf"].v, 0.0); prl.e[F] = np.where(inb, r["rhs_lhs_pdf"].e, 0.0)
    pts = hit_point_f32(r["n2w"], w, r["h"], r["depth"])
    ra = di_ray_f32(r["lhs_point"], pts[(r["rhs_idx"] - 1) // w, (r["rhs_idx"] - 1) % w])
    rb = di_ray_f32(r["rhs_point"], pts[gy[F], lx[F]])
    va = np.where(r["zero_a"], 1.0, 1.0 - np.asarray(trace_any(ra), np.float64))
    vb = np.where(r["zero_b"], 1.0, 1.0 - np.asarray(trace_any(rb), np.float64))
    vis_a[F], vis_b[F] = va, np.where(inb, vb, 0.0)
    skip = r["undecided"].copy()
    traced_a = rhs_idx > 0
    traced_b = traced_a & ((gx * 2 + 1) < w)
    return dict(rhs_idx=rhs_idx, vis_a=vis_a, vis_b=vis_b, lhs_rhs_pdf=plr, rhs_lhs_pdf=prl, skip=skip, traced_a=traced_a & ~skip,
                traced_b=traced_b & ~skip)


def flip_visibility(st, a, b):
    """The composed K9 inputs with the visibility of ray a and / or ray b flipped on every traced pair."""
    out = dict(st)
    if a:
        out["vis_a"] = np.where(st["traced_a"], 1.0 - st["vis_a"], st["vis_a"])
    if b:
        out["vis_b"] = np.where(st["traced_b"], 1.0 - st["vis_b"], st["vis_b"])
    return out


def pick_tight_ok(acc):
    """At least 99 % of K7's finite nonzero lengths and pdfs are bounded below 1e-3 relative."""
    return acc[1] > 0 and acc[0] >= 0.99 * acc[1]


# ---- checks shared by the CPU chain test and the GPU tests --------------------------------------------------------------------

def merge_alternatives(rs):
    """One K9 restatement whose candidates are those of all of `rs` (the same pairs under different visibility bits)."""
    return dict(rs[0], cands=[c for r in rs for c in r["cands"]], undecided=np.logical_or.reduce([r["undecided"] for r in rs]))


def check_spatial_sample(got, res_in, r, what):
    """Every merged pair (but the skipped ones) matches one of its admissible outcomes: the discrete words bit for bit, m, w and a
    bounded pdf within their bounds; the pass-through pixels are copies.  Returns (largest error / bound ratio, undecided pairs,
    merged pairs, visibility bits flipped: the fewest flipped rays any matching candidate needs, summed over the pairs)."""
    got = np.asarray(got, np.float32).reshape(-1, 8)
    g = got[r["idx"]]
    gb = g.view(np.uint32)
    ok = r["skip"].copy()
    best = np.full(len(g), np.inf)
    flips = np.full(len(g), np.inf)
    for c in r["cands"]:
        wb = c["words"].view(np.uint32)
        disc = (gb[:, 3:8] == wb[:, 3:8]).all(1)
        if "pdf" not in c:          # pass-through: every word as read
            ratio = np.where((gb == wb).all(1), 0.0, np.inf)
        else:
            with np.errstate(invalid="ignore", divide="ignore"):
                rat = []
                for k, key in ((0, "m"), (1, "w"), (2, "pdf")):
                    err = np.abs(g[:, k].astype(np.float64) - c[key])
                    rk = np.where(err == 0, 0.0, err / c[key + "_e"])
                    rat.append(np.where(np.isnan(rk), np.inf, rk))
                # an exact pdf (e = 0) is compared bit for bit
                rat[2] = np.where(c["pdf_e"] == 0, np.where(gb[:, 2] == wb[:, 2], 0.0, np.inf), rat[2])
                ratio = np.maximum(np.maximum(rat[0], rat[1]), rat[2])
        good = c["allowed"] & disc & (ratio <= 1.0) & ~r["skip"]
        best = np.where(good, np.minimum(best, ratio), best)
        flips = np.where(good, np.minimum(flips, c["flips"]), flips)
        ok |= good
    if not ok.all():
        i = np.flatnonzero(~ok)[:4]
        raise AssertionError(f"{what}: {int((~ok).sum())}/{len(ok)} pairs match no admissible outcome; first pixels {r['idx'][i].tolist()}: "
                             f"got {g[i].tolist()}")
    cp = r["copies"]
    src = np.asarray(res_in, np.float32).reshape(-1, 8)[cp].view(np.uint32)
    assert (got[cp].view(np.uint32) == src).all(), f"{what}: pass-through reservoirs differ"
    best = best[~r["skip"]]
    flipped = np.where(np.isfinite(flips) & ~r["skip"], flips, 0)
    return (float(best.max()) if len(best) else 0.0, int(r["undecided"].sum()), int((r["merge"] & ~r["skip"]).sum()), int(flipped.sum()))


def spatial_sample_tight(r):
    """(fraction of the merged pairs' finite nonzero m and w whose bound is below 1e-3 of the value, count), over the outcome the f64
    decisions select (undecided pairs are left out)."""
    n = t = 0
    for c in r["cands"]:
        if "pdf" not in c or c["flips"]:
            continue
        sel = c["allowed"] & ~r["undecided"] & ~r["skip"]
        for key in ("m", "w"):
            v, e = c[key][sel], c[key + "_e"][sel]
            fin = np.isfinite(v) & (v != 0)
            n += int(fin.sum()); t += int((e[fin] < 1e-3 * np.abs(v[fin])).sum())
    return t / max(n, 1), n


def check_resolving(diff, spec, res_out, r, what, check_within):
    """K10's outputs at surface pixels against the restatement; the reservoir copy everywhere.  Returns (ratio, undecided, bounds)."""
    some = r["some"]
    diff = np.asarray(diff, np.float32); spec = np.asarray(spec, np.float32)
    assert (np.asarray(res_out, np.float32).reshape(-1, 8).view(np.uint32) == r["res"].view(np.uint32)).all(), f"{what}: reservoir copy"
    assert (diff[..., 3][some] == r["conf"][some]).all() and (spec[..., 3][some] == r["conf"][some]).all(), f"{what}: confidence"
    assert (diff[..., 3][~some] == 1).all() and (spec[..., 3][~some] == 1).all(), f"{what}: sky confidence"
    ratio = check_within(diff[..., :3][some], r["diff"].v[some], r["diff"].e[some], f"{what} diffuse")
    und = r["undecided"]
    took_zero = und[..., None] & (spec[..., :3] == 0)
    want = np.where(took_zero, 0.0, r["spec"].v)
    bound = np.where(took_zero, 0.0, r["spec"].e)
    ratio = max(ratio, check_within(spec[..., :3][some], want[some], bound[some], f"{what} specular"))
    sky = r["sky"]
    ok = sky["domain"]
    assert (spec[..., :3][~some][ok].view(np.uint32) == 0).all(), f"{what}: sky specular is not +0"
    ratio = max(ratio, check_within(diff[..., :3][~some][ok], sky["diff"].v[ok], sky["diff"].e[ok], f"{what} sky"))
    return ratio, int(und.sum()), (r["diff"], r["spec"])


def tight_fraction(nums, some):
    """Fraction of the finite nonzero values of `nums` (list of Num) whose bound is below 1e-3 of the value."""
    n = t = 0
    for x in nums:
        v, e = x.v[some], x.e[some]
        fin = np.isfinite(v) & (v != 0)
        n += int(fin.sum())
        t += int((e[fin] < 1e-3 * np.abs(v[fin])).sum())
    return t / max(n, 1), n


# ---- the sky: Atmosphere::sample -------------------------------------------------------------------------------------------------
# Atmosphere::sample (atmosphere.rs:86-205), World::sun_dir (world.rs:19-25), Ray::intersect_sphere (ray.rs:304-321).  The LUTs are
# read from the engine as exact inputs; the port fetches them with an explicit f32 bilinear filter, clamp to edge, texel centres at
# +0.5.  The fetched value is bounded through its sensitivity to the coordinates: the largest difference of neighbouring texels over
# every cell the coordinates' bounds reach, times those bounds, plus 24 u of the largest texel for the two lerps' roundings.  acos
# near +-1 and sqrt(|altitude|) near the horizon have unbounded derivatives: acos takes its modulus of continuity acos(1 - d) where
# that is smaller than the derivative bound, and Num.sqrt already takes sqrt(e) there.  Four decisions: the nadir branch
# |altitude| > pi / 2 - 1e-4 (altitude is horizon - zenith angle, so the branch is taken looking straight down), the atan2 cut (u
# jumps between 0 and 1 opposite the sun), the sun disc cos >= min_cos and the ground test ray_sphere >= 0.  Where one is within its
# bound, both outcomes are computed and the value is accepted anywhere between them (their hull); the pixel is counted.
ACOS_ABS = 2.0 ** -21           # the strict Cephes acosf on [-1, 1], absolute: 3.0e-7 measured (test_ref64_constants)
ATAN2_ABS = 2.0 ** -21          # the strict Cephes atan2f, absolute: 2.7e-7 measured (test_ref64_constants)
# the fast build runs the same Cephes kernels with FMA contraction, sqrt.approx and div.full inside: measured on an H100, acos 3.2e-7
# and atan2 2.9e-7 (test_fast_elementary_functions_within_assumed_constants).  Inlined into a pass, the compiler may contract them
# differently, each change moving the result by a few of its ulps (<= 2^-22 on results <= pi), so the constant is four times the
# strict one
ACOS_ABS_FAST = ATAN2_ABS_FAST = 2.0 ** -19
ATM_GROUND, ATM_TOP = _f32c(6.360), _f32c(6.460)
ATM_VIEW_Y = _f32c(np.float32(6.360) + np.float32(0.0002))
ATM_ZENITH = _f32c(np.float32(0.5 * np.float32(np.pi)) - np.float32(0.0001))
ATM_EXPOSURE = 20.0
# misreadings of atmosphere.rs that the sky check must catch (test_restir_gi_reference.py)
SKY_MUTATIONS = ("sky_azimuth_no_pi", "sky_altitude_no_sqrt")
SKY_BRANCHES = ("sun disc", "bloom", "ground", "nadir", "atan2 cut")


def atmosphere_inputs(engine):
    """What Atmosphere::sample reads from an engine (the CUDA engine or the oracle): the sky LUT (256 x 256), the transmittance LUT
    (256 x 64) and the sun's (azimuth, altitude)."""
    world = engine.read_scene("world")
    return dict(sky=engine.read_scene("sky_lut").reshape(256, 256, 4), trans=engine.read_scene("transmittance_lut").reshape(64, 256, 4),
                sun=(float(world[1]), float(world[2])))


def cross3(a, b):
    """glam Vec3::cross."""
    ax, ay, az, bx, by, bz = a.col(0), a.col(1), a.col(2), b.col(0), b.col(1), b.col(2)
    return stack3(ay * bz - az * by, az * bx - ax * bz, ax * by - ay * bx)


def _hull(mask, a, b):
    """Where `mask`, a value that covers both a and b; elsewhere a."""
    lo, hi = np.minimum(a.v - a.e, b.v - b.e), np.maximum(a.v + a.e, b.v + b.e)
    with np.errstate(invalid="ignore"):
        return Num(np.where(mask, (lo + hi) / 2, a.v), np.where(mask, (hi - lo) / 2, a.e), a.fast)


def _acos(x):
    """acos of a Num: 1 / sqrt(1 - (|x| + e)^2) times e, or acos(1 - 2 e) wherever that is smaller (the steepest change of acos over
    an interval of width 2 e is at +-1), plus the function's error.  Returns (Num, domain): domain is False where the f32 argument may
    lie outside [-1, 1] (the device returns NaN there)."""
    k = ACOS_ABS_FAST if x.fast else ACOS_ABS
    with np.errstate(invalid="ignore", divide="ignore"):
        reach = np.abs(x.v) + x.e
        slope = np.where(reach < 1, x.e / np.sqrt(np.maximum(1 - reach * reach, 1e-300)), np.inf)
        modulus = np.arccos(np.clip(1 - 2 * x.e, -1, 1))
        v = np.arccos(np.clip(x.v, -1, 1))
    return Num(v, np.minimum(slope, modulus) + k, x.fast), reach <= 1


def _atan2(y, x):
    """atan2(y, x) + nothing: a move of (x, y) by at most d = ex + ey turns the angle by at most asin(d / r), r = |(x, y)|, away from
    the cut (d >= r: anything), plus the function's error."""
    k = ATAN2_ABS_FAST if x.fast else ATAN2_ABS
    r = np.hypot(x.v, y.v)
    d = x.e + y.e
    with np.errstate(invalid="ignore", divide="ignore"):
        turn = np.where(d < r, np.arcsin(np.minimum(d / np.where(r > 0, r, 1.0), 1.0)), np.pi)
    return Num(np.arctan2(y.v, x.v), turn + k, x.fast)


def _exp(x):
    """exp of a Num <= 0: exp(x + e) e for the argument's bound, plus the tier's relative error (R.EXP_REL strict; EXP_REL_FAST and
    __expf's scaled argument in the fast build)."""
    from tests.ref64_svgf import EXP_REL
    rel = (EXP_REL_FAST + 2 * U * np.abs(x.v) * np.log2(np.e)) if x.fast else EXP_REL
    with np.errstate(over="ignore"):
        v = np.exp(x.v)
        return Num(v, np.exp(x.v + x.e) * x.e + rel * v + SUB, x.fast)


def lut_fetch(lut, fx, fy):
    """The port's bilinear fetch of an (H, W, 4) LUT at texel coordinates fx = u W - 0.5, fy = v H - 0.5 (Num (N,)): the exact
    bilinear value at the coordinates' values (clamped to the edge texels' centres), bounded by the coordinates' bounds times the
    largest neighbouring-texel difference over the cells they reach, plus the lerps' roundings.  Returns Num (N, 3)."""
    h, w = lut.shape[:2]
    L = np.asarray(lut, np.float32)[..., :3].astype(np.float64)
    fin = np.isfinite(fx.v) & np.isfinite(fy.v)
    x = np.clip(np.where(fin, fx.v, 0.0), 0, w - 1); y = np.clip(np.where(fin, fy.v, 0.0), 0, h - 1)
    x0 = np.minimum(np.floor(x), w - 2).astype(np.int64); y0 = np.minimum(np.floor(y), h - 2).astype(np.int64)
    tx, ty = (x - x0)[:, None], (y - y0)[:, None]
    a, b, c, d = L[y0, x0], L[y0, x0 + 1], L[y0 + 1, x0], L[y0 + 1, x0 + 1]
    top, bot = a + (b - a) * tx, c + (d - c) * tx
    val = top + (bot - top) * ty
    dx, dy = np.abs(np.diff(L, axis=1)), np.abs(np.diff(L, axis=0))      # (H, W-1, 3), (H-1, W, 3)
    absl = np.abs(L)
    ex, ey = np.where(fin, fx.e, np.inf), np.where(fin, fy.e, np.inf)
    with np.errstate(invalid="ignore"):
        xl = np.clip(np.floor(np.where(fin, fx.v - ex, 0.0)), 0, w - 1).astype(np.int64)
        yl = np.clip(np.floor(np.where(fin, fy.v - ey, 0.0)), 0, h - 1).astype(np.int64)
    # coordinate bounds below one texel reach cells xl..xl+2 and yl..yl+2: the x differences of rows yl..yl+3, the y differences of
    # columns xl..xl+3 (indices clipped to the LUT: a repeated entry only repeats a maximum)
    def win(arr, r, c):
        p = np.pad(arr, ((0, r - 1), (0, c - 1), (0, 0)), mode="edge")
        mx = np.max([p[i:i + arr.shape[0], j:j + arr.shape[1]] for i in range(r) for j in range(c)], axis=0)
        return mx[np.minimum(yl, arr.shape[0] - 1), np.minimum(xl, arr.shape[1] - 1)]
    lx, ly, m = win(dx, 4, 3), win(dy, 3, 4), win(absl, 4, 4)
    err = lx * ex[:, None] + ly * ey[:, None] + 24 * U * m
    for i in np.flatnonzero(~((ex < 1) & (ey < 1))):
        if not (np.isfinite(ex[i]) and np.isfinite(ey[i])):
            err[i] = np.inf
            continue
        xh = int(np.clip(np.floor(fx.v[i] + ex[i]), 0, w - 1)); yh = int(np.clip(np.floor(fy.v[i] + ey[i]), 0, h - 1))
        cx = dx[yl[i]:yh + 2, xl[i]:min(xh + 1, w - 1)].reshape(-1, 3)
        cy = dy[yl[i]:min(yh + 1, h - 1), xl[i]:xh + 2].reshape(-1, 3)
        mm = absl[yl[i]:yh + 2, xl[i]:xh + 2].reshape(-1, 3).max(0)
        err[i] = (cx.max(0) if len(cx) else 0.0) * ex[i] + (cy.max(0) if len(cy) else 0.0) * ey[i] + 24 * U * mm
    return Num(val, err, fx.fast)


def world_sun_dir(azimuth, altitude, fast):
    """World::sun_dir: (cos alt sin az, sin alt, -cos alt cos az) through `sincos`."""
    sa, ca = sincos(Num(np.float64(np.float32(altitude)), 0.0, fast))
    sz, cz = sincos(Num(np.float64(np.float32(azimuth)), 0.0, fast))
    return stack3(ca * sz, sa, (-ca) * cz)


def atmosphere_sample(atm, ray_dir, fast, mutation=None):
    """Atmosphere::sample(sun_dir, ray_dir) for ray directions ray_dir (Num (N, 3)), exposure included.  Returns dict(lum (Num (N,
    3)), domain (False where the zenith angle's acos may be NaN: not compared), undecided {decision: mask}, branches {name: count})."""
    n = ray_dir.v.shape[0]
    z = lambda a: Num(np.broadcast_to(np.asarray(a, np.float64), (n,)).copy(), 0.0, fast)
    sun = world_sun_dir(*atm["sun"], fast)
    sun = Num(np.broadcast_to(sun.v, (n, 3)), np.broadcast_to(sun.e, (n, 3)), fast)
    vp = stack3(z(0.0), z(ATM_VIEW_Y), z(0.0))
    height = dot3(vp, vp).sqrt()
    up = vp / height.x3()
    t = (height * height - z(ATM_GROUND) * ATM_GROUND).sqrt() / height
    horizon, _ = _acos(t.clip(-1.0, 1.0))
    zen, domain = _acos(dot3(ray_dir, up))
    altitude = horizon - zen
    und, br = {}, dict.fromkeys(SKY_BRANCHES, 0)
    # sample_sky_lut: the nadir branch, else the azimuth about the sun
    a = altitude.abs()
    nadir = a.v > ATM_ZENITH
    und["nadir"] = np.abs(a.v - ATM_ZENITH) <= a.e
    right = cross3(sun, up)
    forward = cross3(up, right)
    proj = norm3(ray_dir - up * dot3(ray_dir, up).x3())
    s, c = dot3(proj, right), dot3(proj, forward)
    cut = (c.v < 0) & (np.abs(s.v) <= s.e)          # opposite the sun, the sign of sin theta (and so u = 0 or 1) is undecided
    und["atan2 cut"] = cut & ~nadir

    def fetch(az, nadir):
        if mutation != "sky_azimuth_no_pi":
            az = az + PI
        u = where(nadir, z(0.0), az / _f32c(2 * np.float32(np.pi)))
        m = (altitude.abs() * 2.0) / PI
        m = m if mutation == "sky_altitude_no_sqrt" else m.sqrt()
        sign_known = np.abs(altitude.v) > altitude.e
        half = where(sign_known, Num(np.copysign(m.v, altitude.v), m.e, fast), Num(np.zeros(n), m.v + m.e, fast))
        v = 0.5 + 0.5 * half
        return lut_fetch(atm["sky"], u * 256.0 - 0.5, v * 256.0 - 0.5), u

    ang = _atan2(s, c)
    lum, u = fetch(ang, nadir)
    if cut.any():
        lum = _hull(cut[:, None], lum, fetch(Num(-ang.v, ang.e, fast), nadir)[0])
    if und["nadir"].any():
        lum = _hull(und["nadir"][:, None], lum, fetch(ang, ~nadir)[0])
    br["nadir"] = int((nadir & ~und["nadir"]).sum())
    br["atan2 cut"] = int((~nadir & (c.v < 0) & ((u.v < 0.5 / 256) | (u.v > 1 - 0.5 / 256))).sum())
    # evaluate_bloom / interpolate_bloom
    min_cos = sincos(Num(_f32c(0.53), 0.0, fast) * PI / 180.0)[1]
    cos_t = dot3(ray_dir, sun)
    dc = cos_t - min_cos
    disc = dc.v >= 0
    und["sun disc"] = np.abs(dc.v) <= dc.e
    offset = min_cos - cos_t
    gauss = _exp((-offset) * 50000.0) * 0.5
    inv = (1.0 / (0.02 + offset * 300.0)) * 0.01
    bloom = where(disc, z(1.0), gauss + inv)
    bloom = _hull(und["sun disc"], bloom, where(disc, gauss + inv, z(1.0)))

    def smooth(b):
        tt = ((b - 0.002) / (1.0 - z(0.002))).sat()
        return (tt * tt) * (3.0 - 2.0 * tt)
    sl = smooth(bloom)
    # sun_lum.length_squared() > 0, then Ray::intersect_sphere(GROUND) >= 0 from the view position
    lit = sl.v > 0
    lit_und = (sl.v <= sl.e) & (sl.e > 0)
    b = dot3(vp, ray_dir)
    disc_r = b * b - (dot3(vp, vp) - z(ATM_GROUND) * ATM_GROUND)
    ground = (b.v <= 0) & (disc_r.v >= 0)
    und["ground"] = lit & ((np.abs(disc_r.v) <= disc_r.e) | ((np.abs(b.v) <= b.e) & (disc_r.v + disc_r.e >= 0)))
    trans = lut_fetch(atm["trans"], (0.5 + 0.5 * dot3(sun, up)).sat() * 256.0 - 0.5,
                      ((height - ATM_GROUND) / (z(ATM_TOP) - ATM_GROUND)).sat() * 64.0 - 0.5)
    sun_lum = sl.x3() * trans
    zero3 = Num(np.zeros((n, 3)), 0.0, fast)
    out = where(lit & ~ground, sun_lum, zero3)
    out = _hull((und["ground"] | lit_und)[:, None], out, where(ground & ~und["ground"], zero3, sun_lum))
    br["sun disc"] = int((disc & ~und["sun disc"]).sum())
    br["bloom"] = int((~disc & lit & ~lit_und & ~ground & ~und["ground"]).sum())
    br["ground"] = int((lit & ground & ~und["ground"]).sum())
    lum = (lum + out) * ATM_EXPOSURE
    und = {k: v & domain for k, v in und.items()}
    und["acos domain"] = ~domain
    return dict(lum=lum, domain=domain, undecided=und, branches=br)


# ---- fast-tier elementary functions -----------------------------------------------------------------------------------------
# What a bound on a pass that evaluates these in the fast build assumes (PTX ISA / CUDA programming guide limits, with margin), on
# the arguments the ReSTIR kernels pass: angles 2 pi r for r in [0, 1) and the sun's altitude / azimuth (sin / cos), exponents in
# [-100, 0] (the sun bloom), pow bases in (0, 1] with the exponents of the lights and LUTs, sqrt of [0, 1e6], and divisions.
SIN_ABS = 2.0 ** -23            # the strict build's Cephes sinf / cosf on [0, 2 pi], absolute: 7.6e-8 measured (test_ref64_constants)
SIN_ABS_FAST = 2.0 ** -20       # __sincosf on [0, 2 pi], absolute: 2^-21.4 on [-pi, pi] (CUDA guide), 7.1e-7 measured on an H100 for cos
EXP_REL_FAST = 2.0 ** -21       # __expf(x) = ex2.approx(x log2 e), relative, plus 2 u |x| log2 e for the scaled argument
POW_REL_FAST = 2.0 ** -20       # __powf(x, y) = ex2.approx(y lg2.approx(x)), relative, plus 2^-22 |y log2 x| for lg2's absolute error
