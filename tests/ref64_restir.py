"""Float64 restatement of the DI spatial merge (K9) and DI resolving (K10), with a per-value error bound for either arithmetic tier.

Written from the reference's definitions (paths relative to the reference tree), not from the CUDA kernels or the oracle:
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
  min, max, clamp, saturate, |x|   1-Lipschitz: the input bound passes through.
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
Visibility (Ray::intersect) is not restated: K9 takes it from the scratch texels, K10 from the occluded bit it stores.
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
        self.e = np.zeros(self.v.shape) + np.asarray(e, dtype=np.float64)
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
            return Num(r, e + self._sub(r, self.e, o.e), self.fast)

    def __rtruediv__(self, o):
        return self._n(o) / self

    def sqrt(self):
        rel = SQRT_REL_FAST if self.fast else U
        with np.errstate(invalid="ignore", divide="ignore"):
            s = np.sqrt(np.maximum(self.v, 0.0))
            prop = np.where(s > 0, np.minimum(self.e / np.where(s > 0, s, 1.0), np.sqrt(self.e)), np.sqrt(self.e))
            return Num(s, prop + rel * s + self._sub(s, self.e), self.fast)

    def clip(self, lo, hi):
        return Num(np.clip(self.v, lo, hi), self.e, self.fast)

    def sat(self):
        return self.clip(0.0, 1.0)

    def maximum(self, c):
        return Num(np.maximum(self.v, c), self.e, self.fast)

    def minimum(self, c):
        return Num(np.minimum(self.v, c), self.e, self.fast)

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


def camera_ray(n2w, w, h, fast):
    """Camera::ray for every pixel: (origin, dir) as Num (H, W, 3)."""
    m = np.asarray(n2w, np.float64).reshape(4, 4)          # m[c] = column c
    ys, xs = np.mgrid[0:h, 0:w].astype(np.float64)
    z = lambda a: Num(a, 0.0, fast)
    nx = (z(xs + 0.5) * 2.0) / float(w) - 1.0
    ny = -((z(ys + 0.5) * 2.0) / float(h) - 1.0)

    def project(zc):
        r = [z(m[0][k]) * nx for k in range(4)]
        r = [r[k] + z(m[1][k]) * ny for k in range(4)]
        r = [r[k] + z(np.full((h, w), m[2][k])) * zc for k in range(4)]
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


def hit(n2w, w, h, d0, d1, fast):
    """Hit::new(camera.ray(pos), gbuffer): point = origin + dir * (depth - 0.01)."""
    o, d = camera_ray(n2w, w, h, fast)
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


def light_radiance(L, ht):
    """Light::radiance (light.rs:143-207) for per-pixel light records L (..., 28).  Returns dict(radiance, spec, undecided)."""
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
    rad = ((color * f_angle.x3()) * f_dist.x3()) * f_cos.x3()
    return dict(radiance=rad, spec=spec, undecided=und)


# ---- reservoirs -------------------------------------------------------------------------------------------------------------

def di_fields(res):
    """DiReservoir::read of an (N, 8) buffer: m, w, pdf, occluded, confidence, light point (N, 3), light id."""
    r = np.asarray(res, np.float32).reshape(-1, 8)
    b = r[:, 3].view(np.uint32)
    return dict(m=r[:, 0].astype(np.float64), w=r[:, 1].astype(np.float64), pdf=r[:, 2].astype(np.float64),
                occ=(b & 0xFF) > 0, conf=((b >> 8) & 0xFF).astype(np.float64), point=r[:, 4:7].copy(), id=r[:, 7].view(np.uint32).copy())


def di_resolving(n2w, w, h, d0, d1, lights, res_in, res_out, fast):
    """K10 for the pixels with a surface.  `res_in` = the reservoirs it reads (next), `res_out` = what it wrote (prev): the occluded
    bit there is the visibility the kernel traced.  Returns dict(diff, spec (Num (H, W, 3)), conf (H, W), some, undecided, res)
    where `res` is the (N, 8) reservoir copy expected (with the device's visibility)."""
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
    return dict(diff=diff, spec=spec, conf=conf, some=some, undecided=lr["undecided"] & ~occ & some, res=want)


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


def di_spatial_sample(res_in, stash, seed, frame, w, h, fast):
    """K9 on every checkerboard pair.  Returns dict(idx (P,), cands: list of dicts of expected (P, 8) words + bound on m / w, per-pair
    `allowed` mask per candidate; decided (P,) bool; copies (Q,) indices of the pass-through pixels)."""
    res_in = np.asarray(res_in, np.float32).reshape(-1, 8)
    npx = w * h
    stash = np.asarray(stash, np.float32).reshape(h, w, 4)
    hw = 8 * (((w + 7) // 8) // 2)
    gy, gx = np.mgrid[0:h, 0:hw]
    gx, gy = gx.reshape(-1), gy.reshape(-1)
    f2 = frame // 2
    lx = gx * 2 + ((f2 + 1 + gy) % 2)
    ox = gx * 2 + ((f2 + gy) % 2)
    ok = lx < w
    copies = (gy * w + ox)[(ox < w)]
    gx, gy, lx = gx[ok], gy[ok], lx[ok]
    lidx = gy * w + lx
    ax, bx = gx * 2, gx * 2 + 1
    tz = np.zeros((len(gx), 4), np.float32)
    d0 = np.where((ax < w)[:, None], stash[gy, np.minimum(ax, w - 1)], tz)
    d1 = np.where((bx < w)[:, None], stash[gy, np.minimum(bx, w - 1)], tz)
    rhs_idx = d0[:, 1].view(np.uint32).astype(np.int64)
    # K7 writes 0 (no neighbour) or screen index + 1; anything past the frame would make K9 read outside the reservoirs
    assert not ((rhs_idx > 0) & (rhs_idx - 1 >= npx)).any(), "K7 scratch texel holds a neighbour index outside the frame"
    merge = rhs_idx > 0
    lhs = res_in[lidx]
    rhs = res_in[np.where(merge, rhs_idx - 1, 0)]
    z = lambda a: Num(np.asarray(a, np.float64), 0.0, fast)
    lm, lw, lpdf = z(lhs[:, 0]), z(lhs[:, 1]), z(lhs[:, 2])
    rm, rw, rpdf = z(rhs[:, 0]), z(rhs[:, 1]), z(rhs[:, 2])
    lhs_rhs_vis, rhs_lhs_vis = d0[:, 0].astype(np.float64), d1[:, 0].astype(np.float64)
    lhs_rhs_pdf = z(d1[:, 1]) * lhs_rhs_vis
    rhs_lhs_pdf = z(d1[:, 2]) * rhs_lhs_vis
    with np.errstate(invalid="ignore", over="ignore"):
        mm_a, mm_b = _mis_m(rpdf, rhs_lhs_pdf), _mis_m(lhs_rhs_pdf, lpdf)
        mmin = where(mm_a.v <= mm_b.v, mm_a, mm_b)
        mmin = Num(mmin.v, np.maximum(mm_a.e, mm_b.e), fast)
        mis_m = rm * mmin
        t = _ratio(lm, rm)
        lhs_mis = t + (1.0 - t) * _ratio(lm * lpdf, rm * lhs_rhs_pdf)
        rhs_mis = (1.0 - t) * _ratio((rm * rpdf) * 1.0, lm * rhs_lhs_pdf)
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
            pdf = (rhs_lhs_pdf.v if a2 else (lpdf.v if a1 else np.zeros(len(gx)))).astype(np.float32)
            occ = (lhs_rhs_vis == 0) if a2 else ((src[:, 3].view(np.uint32) & 0xFF) > 0)
            conf = (src[:, 3].view(np.uint32) >> 8) & 0xFF
            with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
                wn = W2 / Num(pdf.astype(np.float64), 0.0, fast)
            wv = np.where(pdf == 0, 0.0, wn.v)
            we = np.where(pdf == 0, 0.0, wn.e)
            out[:, 2] = pdf
            out[:, 3] = (occ.astype(np.uint32) | (conf.astype(np.uint32) << 8)).view(np.float32)
            out[:, 4:8] = src[:, 4:8]
            cands.append(dict(allowed=allowed, words=out, m=m_out.v, m_e=m_out.e, w=wv, w_e=we))
    # no merge: the lhs reservoir goes through as it is
    cands.append(dict(allowed=~merge, words=lhs.copy(), m=lhs[:, 0].astype(np.float64), m_e=np.zeros(len(gx)),
                      w=lhs[:, 1].astype(np.float64), w_e=np.zeros(len(gx))))
    return dict(idx=lidx, cands=cands, undecided=merge & ~(dec1 & dec2), merge=merge, copies=copies)


# ---- checks shared by the CPU chain test and the GPU tests --------------------------------------------------------------------

def check_spatial_sample(got, res_in, r, what):
    """Every merged pair matches one of its admissible outcomes: the discrete words bit for bit, m and w within their bounds; the
    pass-through pixels are copies.  Returns (largest error / bound ratio, undecided pairs, merged pairs)."""
    got = np.asarray(got, np.float32).reshape(-1, 8)
    g = got[r["idx"]]
    gb = g.view(np.uint32)
    ok = np.zeros(len(g), bool)
    best = np.full(len(g), np.inf)
    for c in r["cands"]:
        wb = c["words"].view(np.uint32)
        disc = (gb[:, 2:8] == wb[:, 2:8]).all(1)
        if c is r["cands"][-1]:          # pass-through: every word as read
            ratio = np.where((gb == wb).all(1), 0.0, np.inf)
        else:
            with np.errstate(invalid="ignore", divide="ignore"):
                rat = []
                for k, key in ((0, "m"), (1, "w")):
                    err = np.abs(g[:, k].astype(np.float64) - c[key])
                    rk = np.where(err == 0, 0.0, err / c[key + "_e"])
                    rat.append(np.where(np.isnan(rk), np.inf, rk))
                ratio = np.maximum(rat[0], rat[1])
        good = c["allowed"] & disc & (ratio <= 1.0)
        best = np.where(good, np.minimum(best, ratio), best)
        ok |= good
    if not ok.all():
        i = np.flatnonzero(~ok)[:4]
        raise AssertionError(f"{what}: {int((~ok).sum())}/{len(ok)} pairs match no admissible outcome; first pixels {r['idx'][i].tolist()}: "
                             f"got {g[i].tolist()}")
    cp = r["copies"]
    src = np.asarray(res_in, np.float32).reshape(-1, 8)[cp].view(np.uint32)
    assert (got[cp].view(np.uint32) == src).all(), f"{what}: pass-through reservoirs differ"
    return float(best.max()) if len(best) else 0.0, int(r["undecided"].sum()), int(r["merge"].sum())


def spatial_sample_tight(r):
    """(fraction of the merged pairs' finite nonzero m and w whose bound is below 1e-3 of the value, count), over the outcome the f64
    decisions select (undecided pairs are left out)."""
    n = t = 0
    for c in r["cands"][:-1]:
        sel = c["allowed"] & ~r["undecided"]
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


# ---- fast-tier elementary functions -----------------------------------------------------------------------------------------
# What a bound on a pass that evaluates these in the fast build assumes (PTX ISA / CUDA programming guide limits, with margin), on
# the arguments the ReSTIR kernels pass: angles 2 pi r for r in [0, 1) and the sun's altitude / azimuth (sin / cos), exponents in
# [-100, 0] (the sun bloom), pow bases in (0, 1] with the exponents of the lights and LUTs, sqrt of [0, 1e6], and divisions.
SIN_ABS_FAST = 2.0 ** -20       # __sincosf on [0, 2 pi], absolute: 2^-21.4 on [-pi, pi] (CUDA guide), 7.1e-7 measured on an H100 for cos
EXP_REL_FAST = 2.0 ** -21       # __expf(x) = ex2.approx(x log2 e), relative, plus 2 u |x| log2 e for the scaled argument
POW_REL_FAST = 2.0 ** -20       # __powf(x, y) = ex2.approx(y lg2.approx(x)), relative, plus 2^-22 |y log2 x| for lg2's absolute error
