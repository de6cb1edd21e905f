// ORACLE EXTENSION — TEST INFRASTRUCTURE ONLY.  The environment map (st_set_environment_map) for the CPU oracle.
//
// The oracle in oracle/ restates the reference, whose only sky is the procedural atmosphere, and stays exactly as it is.  This library
// is that oracle (oracle.cpp compiled unchanged into this translation unit) plus the rule of DESIGN.md §2 "Environment map" in the
// oracle's own arithmetic (-ffp-contract=off: every operation one IEEE-754 binary32 operation, in source order):
//   - acos_x / atan2_x (the device's st_device_math ops 8 and 9) and the lookup env_sample;
//   - restatements of the three passes whose sky term changes: K10 (di_resolving), K13 (gi_sampling_b) and K2 (ref_shading), with
//     the map in place of atmosphere_sample and K13's sky-draw probability no longer tied to the sun;
//   - a probe: per evaluated direction, the f32 direction, u, v, the chosen texels and the pass's values around it, for the float64
//     restatement (tests/ref64_envmap.py);
//   - ST_OPT_ENVIRONMENT_MAP_SAMPLING (DESIGN.md §2 "Environment map sampling"): the distribution, env_draw / env_pdf, K12's one-sample
//     mixture and K13's sky draw from the map.
// oracle_envmap/pyoracle_envmap.py steps a frame pass by pass and runs these in place of the oracle's passes while a map is set.
#include "../oracle/oracle.cpp"

namespace {
using namespace orc;

// Test-only mistakes (tests/test_environment_map.py shows that the checks catch each): 0 = the rule.
enum { MUT_NONE = 0, MUT_V_FLIP = 1, MUT_PHI_ZX = 2, MUT_ROT_SIGN = 3, MUT_CLAMP_SEAM = 4, MUT_NO_HALF = 5, MUT_NO_INTENSITY = 6,
       MUT_EXPOSURE = 7, MUT_SUN_GATE = 8,
       // of the sampling (tests/test_environment_map_sampling.py)
       MUT_NO_MAX3 = 9, MUT_NO_SIN_WEIGHT = 10, MUT_NO_SIN_PDF = 11, MUT_DRAW_ROT_SIGN = 12, MUT_COMPONENT_PDF = 13, MUT_NO_KAPPA = 14,
       MUT_DRAW_V_FLIP = 15 };

struct EnvM {
    std::vector<V4> texels; u32 w = 0, h = 0; float intensity = 0.0f, rotation = 0.0f;
    // ST_OPT_ENVIRONMENT_MAP_SAMPLING: the marginal CDF then the conditional CDFs (empty: none built), the marginal's last value, and
    // whether K12 / K13 draw from it (built, and the total finite and > 0)
    std::vector<float> cdf; float total = 0.0f; bool sampled = false;
};

// acos_det / atan2_det's Cephes kernels (st_device.cuh acos_x / atan2_x)
float asin_core_x(float x) {
    const float z = x * x;
    float p = 4.2163199048e-2f;
    p = p * z + 2.4181311049e-2f; p = p * z + 4.5470025998e-2f; p = p * z + 7.4953002686e-2f; p = p * z + 1.6666752422e-1f;
    return (p * z) * x + x;
}
const float HALF_PI_F = 1.5707963267948966f;
float acos_x(float x) {
    if (!(x == x)) return x;
    if (x < -1.0f || x > 1.0f) return u2f(0x7fc00000u);
    if (x > 0.5f) return 2.0f * asin_core_x(sqrtf(0.5f * (1.0f - x)));
    if (x < -0.5f) return PI - 2.0f * asin_core_x(sqrtf(0.5f * (1.0f + x)));
    if (x >= 0.0f) return HALF_PI_F - asin_core_x(x);
    return HALF_PI_F + asin_core_x(-x);
}
float atan_core_x(float x) {
    float y;
    if (x > 2.414213562373095f) { y = HALF_PI_F; x = -(1.0f / x); }
    else if (x > 0.4142135623730950f) { y = 0.7853981633974483f; x = (x - 1.0f) / (x + 1.0f); }
    else y = 0.0f;
    const float z = x * x;
    float p = 8.05374449538e-2f;
    p = p * z - 1.38776856032e-1f; p = p * z + 1.99777106478e-1f; p = p * z - 3.33329491539e-1f;
    return y + ((p * z) * x + x);
}
float atan2_x(float y, float x) {
    if (!(x == x) || !(y == y)) return u2f(0x7fc00000u);
    if (y == 0.0f) {
        if (x > 0.0f || (x == 0.0f && !(f2u(x) >> 31))) return y;
        return copysign_(PI, y);
    }
    if (x == 0.0f) return copysign_(HALF_PI_F, y);
    float a = atan_core_x(abs_(y) / abs_(x));
    if (x < 0.0f) a = PI - a;
    return copysign_(a, y);
}

struct EnvTrace { float u, v; i32 x0, x1, y0, y1; };
V3 env_sample(const EnvM& em, V3 d, int mutation, EnvTrace* tr) {
    const float theta = acos_x(std::min(std::max(d.y, -1.0f), 1.0f));
    const float phi = mutation == MUT_PHI_ZX ? atan2_x(d.z, d.x) : atan2_x(d.x, -d.z);
    const float rot = mutation == MUT_ROT_SIGN ? -em.rotation : em.rotation;
    const float u = (phi + rot) * 0.15915494309189535f + 0.5f;
    float v = theta * 0.3183098861837907f;
    if (mutation == MUT_V_FLIP) v = 1.0f - v;
    if (tr) { tr->u = u; tr->v = v; tr->x0 = tr->x1 = tr->y0 = tr->y1 = -1; }
    if (!(abs_(u) < F32_INF) || !(abs_(v) < F32_INF)) return v3s(0.0f);
    const float half = mutation == MUT_NO_HALF ? 0.0f : 0.5f;
    const float s = u * (float)em.w - half, t = v * (float)em.h - half;
    const float sx = floorf(s), sy = floorf(t);
    const float tx = s - sx, ty = t - sy;
    const i32 W = (i32)em.w, H = (i32)em.h;
    i32 x0, x1;
    if (mutation == MUT_CLAMP_SEAM) { x0 = std::max(0, std::min(f2i_sat(sx), W - 1)); x1 = std::max(0, std::min(f2i_sat(sx) + 1, W - 1)); }
    else { x0 = f2i_sat(sx) % W; if (x0 < 0) x0 += W; x1 = x0 + 1 == W ? 0 : x0 + 1; }
    const i32 iy = f2i_sat(sy);
    const i32 y0 = std::max(0, std::min(iy, H - 1)), y1 = std::max(0, std::min(iy + 1, H - 1));
    if (tr) { tr->x0 = x0; tr->x1 = x1; tr->y0 = y0; tr->y1 = y1; }
    const V3 a = xyz(em.texels[(size_t)y0 * W + x0]), b = xyz(em.texels[(size_t)y0 * W + x1]);
    const V3 c = xyz(em.texels[(size_t)y1 * W + x0]), e = xyz(em.texels[(size_t)y1 * W + x1]);
    const V3 top = a + (b - a) * tx, bot = c + (e - c) * tx;
    V3 r = top + (bot - top) * ty;
    if (mutation != MUT_NO_INTENSITY) r = r * em.intensity;
    if (mutation == MUT_EXPOSURE) r = r * 20.0f;
    return r;
}

// The probe: PROBE_WORDS floats per evaluated direction (tests/ref64_envmap.py reads them).
//   0 site (0 K10 sky pixel, 1 K13 bounce that missed, 2 K13 bounce hit, 3 K2 path that left the scene), 1 pixel index (bits),
//   2-4 the direction, 5 u, 6 v, 7-9 the map's value (0 at a K13 hit that drew a light), 10 K13: the sky-or-light draw (-1 without
//   lights), 11 K13: 1 = the sky was drawn, 12-14 K13: the hit's normal, K2: the throughput, 15 K13: the visibility, 16-18 K13: the
//   hit's base colour, K2: the colour before, 19-21 K13: the hit's emissive, 22-24 the pass's result (K10: the diffuse sample, K13:
//   the radiance, K2: the colour after), 25-27 K10: the specular sample, 28-31 the texel columns x0, x1 and rows y0, y1 (-1: none).
const int PROBE_WORDS = 32;
struct Probe { std::vector<float>* out = nullptr; };
Probe g_probe;
void probe_push(const float* r) {
    if (!g_probe.out) return;
#pragma omp critical(envm_probe)
    g_probe.out->insert(g_probe.out->end(), r, r + PROBE_WORDS);
}
void probe_head(float* r, int site, size_t idx, V3 d, const EnvTrace& tr, V3 env) {
    std::memset(r, 0, sizeof(float) * PROBE_WORDS);
    r[0] = (float)site; r[1] = u2f((u32)idx); r[2] = d.x; r[3] = d.y; r[4] = d.z; r[5] = tr.u; r[6] = tr.v;
    r[7] = env.x; r[8] = env.y; r[9] = env.z;
    r[28] = (float)tr.x0; r[29] = (float)tr.x1; r[30] = (float)tr.y0; r[31] = (float)tr.y1;
}

// ---- ST_OPT_ENVIRONMENT_MAP_SAMPLING ----------------------------------------------------------------------------------------------
// The distribution (kernels.cu k_envdist_rows / k_envdist_marginal): weight = the largest RGB channel over the clamped-row, wrapped-
// column 3x3 neighbourhood times the row's sin(pi (i + 0.5) / H) (double, rounded to f32); f32 running sums in index order.
void envm_build_distribution(EnvM& m, int mutation) {
    const u32 W = m.w, H = m.h;
    m.cdf.assign((size_t)H + (size_t)W * H, 0.0f);
    for (u32 i = 0; i < H; i++) {
        const float st = mutation == MUT_NO_SIN_WEIGHT ? 1.0f : (float)std::sin(3.141592653589793 * ((double)i + 0.5) / (double)H);
        const u32 r0 = i ? i - 1u : 0u, r2 = i + 1u < H ? i + 1u : H - 1u;
        float acc = 0.0f;
        for (u32 j = 0; j < W; j++) {
            const u32 jl = j ? j - 1u : W - 1u, jr = j + 1u < W ? j + 1u : 0u;
            float mx = 0.0f;
            for (u32 r : {r0, i, r2}) {
                if (mutation == MUT_NO_MAX3 && r != i) continue;
                for (u32 c : {jl, j, jr}) {
                    if (mutation == MUT_NO_MAX3 && c != j) continue;
                    const V4 t = m.texels[(size_t)r * W + c];
                    mx = std::max(mx, std::max(std::max(t.x, t.y), t.z));
                }
            }
            acc = acc + mx * st;
            m.cdf[H + (size_t)i * W + j] = acc;
        }
    }
    float acc = 0.0f;
    for (u32 i = 0; i < H; i++) { acc = acc + m.cdf[H + (size_t)i * W + W - 1]; m.cdf[i] = acc; }
    m.total = acc;
}
// st_device.cuh sincos_x
void sincos_x(float xx, float* s_out, float* c_out) {
    float x = abs_(xx);
    u32 j = (u32)(1.27323954473516f * x);
    float y = (float)j;
    if (j & 1u) { j += 1u; y = y + 1.0f; }
    j &= 7u;
    x = ((x - y * 0.78515625f) - y * 2.4187564849853515625e-4f) - y * 3.77489497744594108e-8f;
    const float z = x * x;
    const float ps = ((-1.9515295891e-4f * z + 8.3321608736e-3f) * z - 1.6666654611e-1f) * z * x + x;
    const float pc = ((2.443315711809948e-5f * z - 1.388731625493765e-3f) * z + 4.166664568298827e-2f) * z * z - 0.5f * z + 1.0f;
    float s = (j == 0u) ? ps : (j == 2u) ? pc : (j == 4u) ? -ps : -pc;
    const float c = (j == 0u) ? pc : (j == 2u) ? -ps : (j == 4u) ? -pc : ps;
    if (f2u(xx) & 0x80000000u) s = -s;
    *s_out = s; *c_out = c;
}
u32 env_cdf_find(const float* cdf, u32 n, float t, float last) {
    u32 lo = 0u, hi = n - 1u;
    while (lo < hi) {
        const u32 mid = (lo + hi) >> 1;
        if (cdf[mid] > t || cdf[mid] == last) hi = mid; else lo = mid + 1u;
    }
    return lo;
}
const float BELOW_ONE = 0.99999994039535522f;
// st_device.cuh env_draw; `cell` (optional) receives the drawn row and column
V3 env_draw(const EnvM& em, float xi1, float xi2, int mutation, u32* cell) {
    const u32 W = em.w, H = em.h;
    const float* M = em.cdf.data();
    const float t = xi1 * em.total;
    const u32 i = env_cdf_find(M, H, t, em.total);
    const float m0 = i ? M[i - 1] : 0.0f, m1 = M[i];
    const float dv = std::min((t - m0) / (m1 - m0), BELOW_ONE);
    const float* C = M + H + (size_t)i * W;
    const float rt = C[W - 1];
    const float t2 = xi2 * rt;
    const u32 j = env_cdf_find(C, W, t2, rt);
    const float c0 = j ? C[j - 1] : 0.0f, c1 = C[j];
    const float du = std::min((t2 - c0) / (c1 - c0), BELOW_ONE);
    if (cell) { cell[0] = i; cell[1] = j; }
    const float u = ((float)j + du) / (float)W;
    float v = ((float)i + dv) / (float)H;
    if (mutation == MUT_DRAW_V_FLIP) v = 1.0f - v;
    const float rot = mutation == MUT_DRAW_ROT_SIGN ? -em.rotation : em.rotation;
    const float phi = (u - 0.5f) * 6.283185307179586f - rot, theta = PI * v;
    float st, ct, sp, cp;
    sincos_x(theta, &st, &ct); sincos_x(phi, &sp, &cp);
    return v3(st * sp, ct, -(st * cp));
}
// st_device.cuh env_pdf
float env_pdf(const EnvM& em, V3 d, int mutation) {
    const float theta = acos_x(std::min(std::max(d.y, -1.0f), 1.0f)), phi = atan2_x(d.x, -d.z);
    const float u = (phi + em.rotation) * 0.15915494309189535f + 0.5f, v = theta * 0.3183098861837907f;
    if (!(abs_(u) < F32_INF) || !(abs_(v) < F32_INF)) return 0.0f;
    const i32 W = (i32)em.w, H = (i32)em.h;
    i32 j = f2i_sat(floorf(u * (float)W)) % W; if (j < 0) j += W;
    const i32 i = std::max(0, std::min(f2i_sat(floorf(v * (float)H)), H - 1));
    const float* M = em.cdf.data();
    const float* C = M + H + (size_t)i * W;
    const float pr = M[i] - (i ? M[i - 1] : 0.0f), pc = C[j] - (j ? C[j - 1] : 0.0f);
    if (!(pr > 0.0f) || !(pc > 0.0f)) return 0.0f;
    float st = sqrtf(std::max(0.0f, 1.0f - d.y * d.y));
    if (mutation == MUT_NO_SIN_PDF) st = 1.0f;
    if (st == 0.0f) return F32_INF;
    const float prob = (pr / em.total) * (pc / C[W - 1]);
    return (prob * ((float)W * (float)H)) / (19.739208802178716f * st);
}
float dotx(V3 a, V3 b) { return (a.x * b.x + a.y * b.y) + a.z * b.z; }
V3 normx(V3 a) { const float k = 1.0f / sqrtf(dotx(a, a)); return v3(a.x * k, a.y * k, a.z * k); }
// st_device.cuh env_mixture_pdf (q / kappa); `drawn_env`: which component drew w (for MUT_COMPONENT_PDF)
float env_mixture_pdf(const EnvM& em, const GBufferEntry& g, V3 v, V3 w, int mutation, int drawn_env) {
    const float m = g.metallic;
    const V3 n = g.normal;
    const bool up = dotx(n, w) > 0.0f;
    float pg = 0.0f;
    if (m > 0.0f) {
        const float a = clampf(g.roughness, 0.089f * 0.089f, 1.0f), a2 = a * a;
        const V3 h = normx(v3(w.x + v.x, w.y + v.y, w.z + v.z));
        const float n_dot_h = clampf(dotx(n, h), 0.0f, 1.0f), h_dot_v = clampf(dotx(h, v), 0.0f, 1.0f);
        if (n_dot_h > 0.0f && h_dot_v > 0.0f) {
            const float dd = (n_dot_h * a2 - n_dot_h) * n_dot_h + 1.0f;
            const float dist = a2 / ((PI * dd) * dd);
            pg = (dist * n_dot_h) / (4.0f * h_dot_v);
        }
    }
    const float om = 1.0f - m;
    float kappa = (up ? (om * om) * 0.5f : 0.0f) + (pg > 0.0f ? m * m : 0.0f);
    if (mutation == MUT_NO_KAPPA) kappa = 1.0f;
    if (!(kappa > 0.0f)) return F32_INF;
    const float pb = (up ? om * 0.15915494309189535f : 0.0f) + m * pg;
    const float pe = env_pdf(em, w, mutation);
    float q = 0.5f * pb + 0.5f * pe;
    if (mutation == MUT_COMPONENT_PDF) q = drawn_env ? 0.5f * pe : 0.5f * pb;
    return q / kappa;
}
// K12's bounce direction under ENV_SAMPLED (kernels.cu gi_sampling_a_pair): returns q / kappa, the direction in *dir
float env_k12_draw(const EnvM& em, const GBufferEntry& g, V3 v, WhiteNoise& wn, int mutation, V3* dir) {
    int drawn_env;
    if (wnoise_sample(wn) < 0.5f) { const float xi1 = wnoise_sample(wn), xi2 = wnoise_sample(wn); *dir = env_draw(em, xi1, xi2, mutation, nullptr); drawn_env = 1; }
    else { *dir = layered_brdf_sample(g, wn, v).dir; drawn_env = 0; }
    return env_mixture_pdf(em, g, v, *dir, mutation, drawn_env);
}
// K13's sky draw under ENV_SAMPLED: the value L max(n.w, 0) / (2 pi p_env) (before the 1 / 0.25), the direction in *dir, *below = no
// shadow ray
V3 env_k13_sky(const EnvM& em, V3 n, WhiteNoise& wn, int mutation, V3* dir, bool* below) {
    const float xi1 = wnoise_sample(wn), xi2 = wnoise_sample(wn);
    *dir = env_draw(em, xi1, xi2, mutation, nullptr);
    const float c = dotx(n, *dir);
    *below = !(c > 0.0f);
    const float p = *below ? 0.0f : env_pdf(em, *dir, mutation);
    if (!(p > 0.0f)) return v3s(0.0f);
    const V3 l = env_sample(em, *dir, 0, nullptr);
    const float k = c / (6.283185307179586f * p);
    return v3(l.x * k, l.y * k, l.z * k);
}

// K12 (orc_passes.hpp pass_gi_sampling_a) with the one-sample mixture on tracing frames
void envm_gi_sampling_a(CamState& cs, const Scene& sc, const EnvM& em, bool alternate, u32 seed, u32 frame, int mutation) {
    int cur = alternate ? 1 : 0;
    const Camera& cam = cs.curr_camera;
    bool tracing = frame_is_gi_tracing(frame);
    ORC_FOR_HALF_GRID(cs) {
        UV2 gid = uv2(gx_, gy_);
        UV2 sp = tracing ? resolve_checkerboard(gid, frame / 2) : resolve_checkerboard(gid, frame);
        size_t idx = camera_screen_to_idx(cam, sp);
        if (!camera_contains(cam, sp)) continue;
        Ray gi_ray; float gi_ray_pdf;
        if (tracing) {
            WhiteNoise wn = wnoise_new(seed, sp);
            Hit hit = load_hit(cam, cs.prim_gbuffer_d0[cur], cs.prim_gbuffer_d1[cur], cs.w, sp);
            if (!hit_is_some(hit)) continue;
            V3 dir;
            gi_ray_pdf = env_k12_draw(em, hit.gbuffer, -hit.dir, wn, mutation, &dir);
            gi_ray = ray_new(hit.point, dir);
        } else {
            GiReservoir res = gi_read(cs.gi_reservoirs[2].data(), idx);
            if (gi_is_empty(res)) continue;
            gi_ray = ray_new(res.sample.v1_point, gi_sample_dir(res.sample, res.sample.v1_point));
            gi_ray_pdf = 1.0f;
        }
        TriangleHit gh = ray_trace(gi_ray, sc);
        GBufferEntry gg = gbuffer_default();
        if (trihit_is_some(gh)) {
            Material m = sc.materials[gh.material_id];
            material_regularize(m);
            gg.base_color = material_base_color(sc, m, gh.uv);
            gg.normal = gh.normal; gg.metallic = m.metallic; gg.emissive = material_emissive(sc, m, gh.uv);
            gg.roughness = m.roughness; gg.reflectance = m.reflectance;
            gg.depth = distance(gi_ray.origin, gh.point);
        }
        V4 d1, d2; gbuffer_pack(gg, &d1, &d2);
        at(cs.gi_d0, cs.w, gid) = v4(gi_ray.dir, gi_ray_pdf);
        at(cs.gi_d1, cs.w, gid) = d1;
        at(cs.gi_d2, cs.w, gid) = d2;
    }
}

// K10 (orc_passes.hpp pass_di_resolving) with the map for sky pixels
void envm_di_resolving(CamState& cs, const Scene& sc, const EnvM& em, bool alternate, int mutation) {
    int cur = alternate ? 1 : 0;
    const Camera& cam = cs.curr_camera;
    ORC_FOR_FULL_GRID(cs) {
        UV2 p = uv2(gx_, gy_);
        size_t idx = camera_screen_to_idx(cam, p);
        Hit hit = load_hit(cam, cs.prim_gbuffer_d0[cur], cs.prim_gbuffer_d1[cur], cs.w, p);
        DiReservoir res = di_read(cs.di_reservoirs[2].data(), idx);
        float confidence;
        LightRadiance radiance;
        EnvTrace tr{};
        if (hit_is_some(hit)) {
            bool is_occluded = ray_intersect(di_sample_ray(res.sample, hit.point), sc);
            confidence = (res.sample.is_occluded == is_occluded) ? res.sample.confidence : 0.0f;
            res.sample.confidence = 1.0f;
            res.sample.is_occluded = is_occluded;
            if (is_occluded) radiance = light_radiance_default();
            else { radiance = light_radiance(sc.lights[res.sample.light_id], hit); radiance.radiance *= res.w; }
        } else {
            confidence = 1.0f;
            radiance.radiance = env_sample(em, hit.dir, mutation, &tr);
            radiance.diff_brdf = v3s(1.0f); radiance.spec_brdf = v3s(0.0f);
        }
        float diff_brdf = (1.0f - hit.gbuffer.metallic) / PI;
        const V4 dv = v4(radiance.radiance * diff_brdf, confidence), sv = v4(radiance.radiance * radiance.spec_brdf, confidence);
        at(cs.di_diff_samples, cs.w, p) = dv;
        at(cs.di_spec_samples, cs.w, p) = sv;
        di_write(res, cs.di_reservoirs[0].data(), idx);
        if (!hit_is_some(hit) && g_probe.out) {
            float r[PROBE_WORDS]; probe_head(r, 0, idx, hit.dir, tr, radiance.radiance);
            r[22] = dv.x; r[23] = dv.y; r[24] = dv.z; r[25] = sv.x; r[26] = sv.y; r[27] = sv.z;
            probe_push(r);
        }
    }
}

// K13 (orc_passes.hpp pass_gi_sampling_b) with the map for the missed bounce and the sky draw, whose probability is 0.25 whatever the
// sun's altitude
void envm_gi_sampling_b(CamState& cs, const Scene& sc, const EnvM& em, bool alternate, u32 seed, u32 frame, int mutation) {
    int cur = alternate ? 1 : 0;
    const Camera& cam = cs.curr_camera;
    bool tracing = frame_is_gi_tracing(frame);
    ORC_FOR_HALF_GRID(cs) {
        UV2 gid = uv2(gx_, gy_);
        UV2 sp = tracing ? resolve_checkerboard(gid, frame / 2) : resolve_checkerboard(gid, frame);
        size_t idx = camera_screen_to_idx(cam, sp);
        if (!camera_contains(cam, sp)) continue;
        Hit prim_hit = load_hit(cam, cs.prim_gbuffer_d0[cur], cs.prim_gbuffer_d1[cur], cs.w, sp);
        if (!hit_is_some(prim_hit)) continue;
        V4 d0 = at(cs.gi_d0, cs.w, gid), d1 = at(cs.gi_d1, cs.w, gid), d2 = at(cs.gi_d2, cs.w, gid);
        WhiteNoise wn; Hit gi_hit; float gi_ray_pdf;
        if (tracing) {
            wn = wnoise_new(seed, sp);
            gi_hit = hit_new(ray_new(prim_hit.point, xyz(d0)), gbuffer_unpack(d1, d2));
            gi_ray_pdf = d0.w;
        } else {
            GiReservoir res = gi_read(cs.gi_reservoirs[2].data(), idx);
            if (gi_is_empty(res)) continue;
            wn.state = res.sample.rng;
            gi_hit = hit_new(ray_new(res.sample.v1_point, xyz(d0)), gbuffer_unpack(d1, d2));
            gi_ray_pdf = 1.0f;
        }
        u32 rng = wn.state;
        const u32 SKY = 0xffffffffu;
        u32 light_id; float light_pdf; V3 light_rad; V3 light_dir = v3s(0);
        float r[PROBE_WORDS]; EnvTrace tr{-1.0f, -1.0f, -1, -1, -1, -1}; V3 env = v3s(0); float draw = -1.0f;
        bool sky_below = false;   // ST_OPT_ENVIRONMENT_MAP_SAMPLING: the sky draw points below the surface (no shadow ray)
        if (!hit_is_some(gi_hit)) {
            light_id = SKY; light_pdf = 1.0f; light_rad = env = env_sample(em, gi_hit.dir, mutation, &tr);
        } else {
            float atmosphere_pdf = (mutation == MUT_SUN_GATE && sc.world.sun_altitude <= -1.0f) ? 0.0f : 0.25f;
            bool sky;
            if (sc.world.light_count == 0) sky = true;
            else { draw = wnoise_sample(wn); sky = draw < atmosphere_pdf; }
            if (sky && em.sampled) {
                light_id = SKY; light_pdf = atmosphere_pdf;
                light_rad = env_k13_sky(em, gi_hit.gbuffer.normal, wn, mutation, &light_dir, &sky_below);
                env = env_sample(em, light_dir, 0, &tr);
            } else if (sky) {
                light_id = SKY; light_pdf = atmosphere_pdf;
                light_dir = wnoise_sample_hemisphere(wn, gi_hit.gbuffer.normal);
                env = env_sample(em, light_dir, mutation, &tr);
                light_rad = env * dot(gi_hit.gbuffer.normal, light_dir);
            } else {
                EphemeralReservoir res = ephemeral_build(wn, sc, gi_hit);
                if (res.w > 0.0f) {
                    light_id = res.sample.light_id;
                    light_pdf = (1.0f / res.w) * (1.0f - atmosphere_pdf);
                    light_rad = res.sample.light_rad.radiance * (v3s(1.0f) + res.sample.light_rad.spec_brdf);
                } else { light_id = 0; light_pdf = 1.0f; light_rad = v3s(0); }
            }
        }
        V3 radiance;
        float light_vis = 0.0f;
        if (light_pdf > 0.0f) {
            if (hit_is_some(gi_hit)) {
                if (sky_below) light_vis = 0.0f;
                else {
                    Ray ray = (light_id == SKY) ? ray_new(gi_hit.point, light_dir) : light_ray_wnoise(sc.lights[light_id], wn, gi_hit.point);
                    light_vis = ray_intersect(ray, sc) ? 0.0f : 1.0f;
                }
            } else light_vis = 1.0f;
            radiance = light_rad * light_vis / light_pdf;
        } else radiance = v3s(0);
        if (hit_is_some(gi_hit)) {
            radiance *= xyz(gi_hit.gbuffer.base_color) / PI;
            radiance += gi_hit.gbuffer.emissive;
        }
        if (g_probe.out) {
            const bool hit = hit_is_some(gi_hit);
            probe_head(r, hit ? 2 : 1, idx, hit ? light_dir : gi_hit.dir, tr, env);
            if (hit) {
                r[10] = draw; r[11] = light_id == SKY ? 1.0f : 0.0f;
                r[12] = gi_hit.gbuffer.normal.x; r[13] = gi_hit.gbuffer.normal.y; r[14] = gi_hit.gbuffer.normal.z; r[15] = light_vis;
                r[16] = gi_hit.gbuffer.base_color.x; r[17] = gi_hit.gbuffer.base_color.y; r[18] = gi_hit.gbuffer.base_color.z;
                r[19] = gi_hit.gbuffer.emissive.x; r[20] = gi_hit.gbuffer.emissive.y; r[21] = gi_hit.gbuffer.emissive.z;
            }
            r[22] = radiance.x; r[23] = radiance.y; r[24] = radiance.z;
            probe_push(r);
        }
        GiReservoir res = gi_default();
        if (gi_ray_pdf > 0.0f) {
            V3 v1 = prim_hit.point, v2p, v2n;
            if (hit_is_some(gi_hit)) { v2p = gi_hit.point; v2n = gi_hit.gbuffer.normal; }
            else { v2p = v1 + gi_hit.dir * 1000.0f; v2n = -gi_hit.dir; }
            res.sample.pdf = 0.0f; res.sample.rng = rng; res.sample.radiance = radiance;
            res.sample.v1_point = v1; res.sample.v2_point = v2p; res.sample.v2_normal = v2n;
            res.m = 1.0f; res.w = 1.0f / gi_ray_pdf;
            res.sample.pdf = gi_sample_pdf(res.sample, prim_hit);
        }
        gi_write(res, cs.gi_reservoirs[1].data(), idx);
    }
}

// K2 (orc_passes.hpp pass_ref_shading) with the map for a path that leaves the scene; depth < 255 (the accumulation step evaluates
// no sky and stays the oracle's)
void envm_ref_shading(CamState& cs, const Scene& sc, const EnvM& em, u32 seed, u32 depth, int mutation) {
    const Camera& cam = cs.curr_camera;
    ORC_FOR_FULL_GRID(cs) {
        UV2 p = uv2(gx_, gy_);
        size_t idx = camera_screen_to_idx(cam, p);
        WhiteNoise wn = wnoise_new(seed, p);
        V4* rays = cs.ref_rays.data();
        Ray ray; V3 color, throughput;
        if (depth == 0) { ray = camera_ray(cam, p); color = v3s(0); throughput = v3s(1.0f); }
        else {
            V4 d0 = rays[3 * idx], d1 = rays[3 * idx + 1], d2 = rays[3 * idx + 2];
            if (is_zero(d1)) continue;
            ray = ray_new(xyz(d0), xyz(d1)); color = xyz(d2); throughput = v3(d0.w, d1.w, d2.w);
        }
        TriangleHit th = trihit_unpack(cs.ref_hits[2 * idx], cs.ref_hits[2 * idx + 1]);
        if (!trihit_is_some(th)) {
            EnvTrace tr{};
            const V3 env = env_sample(em, ray.dir, mutation, &tr);
            const V3 before = color;
            color += throughput * env;
            rays[3 * idx] = v4z(); rays[3 * idx + 1] = v4z(); rays[3 * idx + 2] = v4(color, 0.0f);
            if (g_probe.out) {
                float r[PROBE_WORDS]; probe_head(r, 3, idx, ray.dir, tr, env);
                r[12] = throughput.x; r[13] = throughput.y; r[14] = throughput.z; r[16] = before.x; r[17] = before.y; r[18] = before.z;
                r[22] = color.x; r[23] = color.y; r[24] = color.z;
                probe_push(r);
            }
            continue;
        }
        Material material = sc.materials[th.material_id];
        if (depth > 0) material_regularize(material);
        Hit hit;
        hit.point = th.point + th.normal * 0.01f; hit.origin = ray.origin; hit.dir = ray.dir;
        hit.gbuffer.base_color = material_base_color(sc, material, th.uv); hit.gbuffer.normal = th.normal; hit.gbuffer.metallic = material.metallic;
        hit.gbuffer.emissive = material_emissive(sc, material, th.uv); hit.gbuffer.roughness = material.roughness;
        hit.gbuffer.reflectance = material.reflectance; hit.gbuffer.depth = 0.0f;
        color += throughput * hit.gbuffer.emissive;
        if (sc.world.light_count > 0) {
            u32 light_id = wnoise_sample_int(wn) % sc.world.light_count;
            float light_pdf = 1.0f / (float)sc.world.light_count;
            const Light& light = sc.lights[light_id];
            bool occluded = ray_intersect(light_ray_wnoise(light, wn, hit.point), sc);
            if (!occluded) color += throughput * light_radiance_sum(light_radiance(light, hit)) / light_pdf;
        }
        BrdfSample rs = layered_brdf_sample(hit.gbuffer, wn, -hit.dir);
        if (rs.pdf == 0.0f) { rays[3 * idx] = v4z(); rays[3 * idx + 1] = v4z(); continue; }
        Ray rr = ray_new(hit.point, rs.dir);
        throughput *= dot(rs.dir, hit.gbuffer.normal);
        throughput *= rs.radiance / rs.pdf;
        rays[3 * idx] = v4(rr.origin, throughput.x);
        rays[3 * idx + 1] = v4(rr.dir, throughput.y);
        rays[3 * idx + 2] = v4(color, throughput.z);
    }
}

}  // namespace

extern "C" {

void* orc_envm_create() { return new EnvM(); }
void orc_envm_destroy(void* m) { delete (EnvM*)m; }
// st_set_environment_map's validation and rotation reduction; 0 = set (or cleared: rgba NULL, returns 1), -1 = invalid (nothing changes)
int orc_envm_set(void* mp, const float* rgba, uint32_t w, uint32_t h, float intensity, float rotation) {
    EnvM& m = *(EnvM*)mp;
    if (!rgba) { m.texels.clear(); m.w = m.h = 0; return 1; }
    if (w < 1u || w > 16384u || h < 1u || h > 16384u || !std::isfinite(intensity) || intensity < 0.0f || !std::isfinite(rotation)) return -1;
    const size_t n = (size_t)w * h;
    for (size_t i = 0; i < n; i++) for (int c = 0; c < 3; c++) if (!std::isfinite(rgba[4 * i + c]) || rgba[4 * i + c] < 0.0f) return -1;
    const double two_pi = 6.283185307179586476925286766559;
    double r = std::fmod((double)rotation, two_pi);
    if (r < 0.0) r += two_pi;
    if (r >= two_pi) r = 0.0;
    m.texels.resize(n); std::memcpy(m.texels.data(), rgba, n * sizeof(V4));
    m.w = w; m.h = h; m.intensity = intensity; m.rotation = (float)r;
    return 0;
}
void orc_envm_copy(void* dst, const void* src) { *(EnvM*)dst = *(const EnvM*)src; }
// st_read_scene("environment_map")'s words; returns the word count (0: no map), copies min(cap, count)
long orc_envm_read(void* mp, float* dst, long cap) {
    const EnvM& m = *(const EnvM*)mp;
    if (m.texels.empty()) return 0;
    std::vector<float> w(4 + 4 * m.texels.size());
    w[0] = u2f(m.w); w[1] = u2f(m.h); w[2] = m.intensity; w[3] = m.rotation;
    std::memcpy(w.data() + 4, m.texels.data(), m.texels.size() * sizeof(V4));
    if (dst) std::memcpy(dst, w.data(), sizeof(float) * (size_t)std::min<long>(cap, (long)w.size()));
    return (long)w.size();
}
// ops 8 (acos_x(a)) and 9 (atan2_x(a, b)) of st_device_math
void orc_envm_math(int op, const float* a, const float* b, float* out, long n) {
    for (long i = 0; i < n; i++) out[i] = op == 8 ? acos_x(a[i]) : atan2_x(a[i], b[i]);
}
// The lookup on its own: out = n x 3 radiances for n directions (3 floats each)
void orc_envm_sample(void* mp, const float* dirs, long n, int mutation, float* out) {
    const EnvM& m = *(const EnvM*)mp;
    for (long i = 0; i < n; i++) {
        const V3 r = env_sample(m, v3(dirs[3 * i], dirs[3 * i + 1], dirs[3 * i + 2]), mutation, nullptr);
        out[3 * i] = r.x; out[3 * i + 1] = r.y; out[3 * i + 2] = r.z;
    }
}
// Runs step `pass` (the device's PassId: 6 = K10, 9 = K13, 22 = K2 at bounce `depth`) of camera `cam`'s current frame with the map,
// in place of the oracle's.  `probe` (optional): receives the probe records (PROBE_WORDS floats each), up to `cap` floats; returns
// the record count, or < 0 on a bad call.
long orc_envm_apply(void* e, void* mp, int cam, int pass, int depth, int mutation, float* probe, long cap) {
    Engine* en = (Engine*)e;
    const EnvM& m = *(const EnvM*)mp;
    if (m.texels.empty()) return -2;
    Engine::Cam* c = en->cameras[cam];
    CamState& cs = c->st;
    en->run_atmosphere();
    const Scene sc = en->scene();
    const u32 f = c->frame;
    const bool alt = (f % 2) == 1;
    std::vector<float> rec;
    g_probe.out = probe ? &rec : nullptr;
    if (pass == 8 && m.sampled) envm_gi_sampling_a(cs, sc, m, alt, dispatch_seed(en->seed_base, f, D_GI_SAMPLING_A), f, mutation);
    else if (pass == 6) envm_di_resolving(cs, sc, m, alt, mutation);
    else if (pass == 9) envm_gi_sampling_b(cs, sc, m, alt, dispatch_seed(en->seed_base, f, D_GI_SAMPLING_B), f, mutation);
    else if (pass == 22 && depth >= 0 && depth < 31) envm_ref_shading(cs, sc, m, dispatch_seed(en->seed_base, f, D_REF_SHADING + (u32)depth), (u32)depth, mutation);
    else { g_probe.out = nullptr; return -1; }
    g_probe.out = nullptr;
    const long n = (long)(rec.size() / PROBE_WORDS);
    if (probe) std::memcpy(probe, rec.data(), sizeof(float) * (size_t)std::min<long>(cap, (long)rec.size()));
    return n;
}

// ST_OPT_ENVIRONMENT_MAP_SAMPLING: on = build the distribution of the map `mp` holds (K12 / K13 then draw from it where its total is
// finite and > 0), off = drop it; returns the total's bits as a float
float orc_envm_distribution(void* mp, int on, int mutation) {
    EnvM& m = *(EnvM*)mp;
    if (!on || m.texels.empty()) { m.cdf.clear(); m.total = 0.0f; m.sampled = false; return 0.0f; }
    envm_build_distribution(m, mutation);
    m.sampled = m.total > 0.0f && m.total < F32_INF;
    return m.total;
}
// st_read_scene("environment_map_distribution")'s words; returns the word count (0: none), copies min(cap, count)
long orc_envm_read_distribution(void* mp, float* dst, long cap) {
    const EnvM& m = *(const EnvM*)mp;
    if (m.cdf.empty()) return 0;
    std::vector<float> w(3 + m.cdf.size());
    w[0] = u2f(m.w); w[1] = u2f(m.h); w[2] = m.total;
    std::memcpy(w.data() + 3, m.cdf.data(), m.cdf.size() * sizeof(float));
    if (dst) std::memcpy(dst, w.data(), sizeof(float) * (size_t)std::min<long>(cap, (long)w.size()));
    return (long)w.size();
}
// env_draw for n (xi1, xi2) pairs: out = n x 3 directions, cells = n x 2 (row, column); env_pdf for n directions
void orc_envm_draw(void* mp, const float* xi, long n, int mutation, float* out, uint32_t* cells) {
    const EnvM& m = *(const EnvM*)mp;
    for (long k = 0; k < n; k++) {
        const V3 d = env_draw(m, xi[2 * k], xi[2 * k + 1], mutation, cells + 2 * k);
        out[3 * k] = d.x; out[3 * k + 1] = d.y; out[3 * k + 2] = d.z;
    }
}
void orc_envm_pdf(void* mp, const float* dirs, long n, int mutation, float* out) {
    const EnvM& m = *(const EnvM*)mp;
    for (long k = 0; k < n; k++) out[k] = env_pdf(m, v3(dirs[3 * k], dirs[3 * k + 1], dirs[3 * k + 2]), mutation);
}
// K12's mixture draw and K13's sky draw at one surface (normal n, view v, metallic, roughness), for n seeds each starting a
// WhiteNoise: out = n x 8 {direction, q / kappa (K12) or p_env (K13), the map's value along the direction}; K13 (`k13` != 0)
// writes the sky-draw value (L max(n.w, 0) / (2 pi p_env)) in place of the map's value and 0 / 1 (below) in word 3
void orc_envm_surface_draws(void* mp, int k13, const float* nvmr, const uint32_t* seeds, long n, int mutation, float* out) {
    const EnvM& m = *(const EnvM*)mp;
    GBufferEntry g = gbuffer_default();
    g.normal = v3(nvmr[0], nvmr[1], nvmr[2]); g.metallic = nvmr[6]; g.roughness = nvmr[7]; g.reflectance = 0.5f;
    g.base_color = v4(1.0f, 1.0f, 1.0f, 1.0f);
    const V3 v = v3(nvmr[3], nvmr[4], nvmr[5]);
    for (long k = 0; k < n; k++) {
        WhiteNoise wn; wn.state = seeds[k];
        V3 d, val; float w;
        if (k13) { bool below; val = env_k13_sky(m, g.normal, wn, mutation, &d, &below); w = below ? 1.0f : 0.0f; }
        else { w = env_k12_draw(m, g, v, wn, mutation, &d); val = env_sample(m, d, 0, nullptr); }
        float* o = out + 8 * k;
        o[0] = d.x; o[1] = d.y; o[2] = d.z; o[3] = w; o[4] = val.x; o[5] = val.y; o[6] = val.z; o[7] = 0.0f;
    }
}

}  // extern "C"
