// ORACLE EXTENSION — TEST INFRASTRUCTURE ONLY.  Texture filtering (ST_OPT_TEXTURE_FILTER) for the CPU oracle.
//
// The oracle in oracle/ restates the reference, whose sampler takes the nearest texel of level 0, and stays exactly as it is.  This
// library is that oracle (oracle.cpp compiled unchanged into this translation unit) plus the rule of DESIGN.md §2 "Texture filtering"
// in the oracle's own arithmetic:
//   - the mip chains (orc_texf_build), laid out as st_read_scene("texture_mips") returns them;
//   - K0 and K12 patches (orc_texf_apply): those passes store the material terms only through gbuffer_pack, so re-tracing the pass's
//     ray (same ray, same BVH: same triangle) and overwriting the packed base colour, emissive and metallic-roughness fields gives
//     exactly what the pass would have stored with the filter;
//   - a restatement of K2 (orc_texf_apply, pass 22) that shades with the filtered terms;
//   - orc_texf_probe: the fetch's inputs and results at every hit, for the float64 restatement.
// oracle_texfilter/pyoracle_texfilter.py steps a frame pass by pass and calls these where the device runs its TEXF kernels.
#include "../oracle/oracle.cpp"

namespace {
using namespace orc;

// Test-only mistakes (tests/test_texture_filter.py shows that the checks catch each): 0 = the rule.
enum { MUT_NONE = 0, MUT_RAW_BYTES = 1, MUT_NO_COS = 2, MUT_CLAMP_ATLAS = 3, MUT_NO_HALF = 4, MUT_SWAP_LEVELS = 5 };

struct TexF {
    std::vector<uint8_t> pool;    // RGBA8 texels
    std::vector<u32> table;       // 2 words per material and colour slot
    size_t texels = 0; u32 materials = 0; bool built = false;
};

float rmax_(float a, float b) { return (a != a) ? b : ((b != b) ? a : (a > b ? a : b)); }
float rclamp_(float x, float lo, float hi) { if (x < lo) x = lo; if (x > hi) x = hi; return x; }
float len3(V3 a) { return sqrtf((a.x * a.x + a.y * a.y) + a.z * a.z); }
V3 cross3(V3 a, V3 b) { return v3(a.y * b.z - b.y * a.z, a.z * b.x - b.z * a.x, a.x * b.y - b.x * a.y); }
float dot3(V3 a, V3 b) { return (a.x * b.x + a.y * b.y) + a.z * b.z; }

// log2_x (st_device.cuh): exponent bits + the Cephes logf polynomial, times log2(e)
float log2_x(float x) {
    u32 bits = f2u(x);
    int e;
    if ((bits & 0x7f800000u) == 0u) { x = x * 8388608.0f; bits = f2u(x); e = (int)((bits >> 23) & 0xffu) - 126 - 23; }
    else e = (int)((bits >> 23) & 0xffu) - 126;
    float m = u2f((bits & 0x007fffffu) | 0x3f000000u);
    if (m < 0.707106781186547524f) { e -= 1; m = (m + m) - 1.0f; } else m = m - 1.0f;
    const float z = m * m;
    float y = 7.0376836292e-2f;
    y = y * m + -1.1514610310e-1f; y = y * m + 1.1676998740e-1f; y = y * m + -1.2420140846e-1f;
    y = y * m + 1.4249322787e-1f; y = y * m + -1.6668057665e-1f; y = y * m + 2.0000714765e-1f;
    y = y * m + -2.4999993993e-1f; y = y * m + 3.3333331174e-1f;
    y = (y * m) * z;
    y = y + -0.5f * z;
    const float ln_m = m + y;
    return ln_m * 1.44269504088896341f + (float)e;
}

void build(TexF& t, const Engine& en, int mutation) {
    struct Chain { u32 x, y, w, h, off1, levels; };
    std::vector<Chain> chains;
    size_t total = 0;
    for (const auto& r : en.images) {
        Chain c = {r.x, r.y, r.w, r.h, (u32)total, 1u};
        for (u32 w = r.w, h = r.h; w > 1u || h > 1u; c.levels++) { w = std::max(1u, w >> 1); h = std::max(1u, h >> 1); total += (size_t)w * h; }
        chains.push_back(c);
    }
    t.texels = total; t.pool.assign(total * 4, 0); t.materials = (u32)en.gpu_materials.size();
    t.table.assign(6 * (size_t)t.materials, 0u);
    for (size_t i = 0; i < en.gpu_materials.size(); i++) {
        const Material& g = en.gpu_materials[i];
        const V4 rects[3] = {g.base_color_texture, g.emissive_texture, g.metallic_roughness_texture};
        for (int k = 0; k < 3; k++) {
            const V4 r = rects[k];
            if (is_zero(r)) continue;
            u32 off = 0, lv = 1;
            for (const Chain& c : chains)
                if (r.x == (float)c.x / (float)ATLAS_SIZE && r.y == (float)c.y / (float)ATLAS_SIZE && r.z == (float)c.w / (float)ATLAS_SIZE && r.w == (float)c.h / (float)ATLAS_SIZE) {
                    off = c.off1; lv = c.levels; break;
                }
            t.table[6 * i + 2 * k] = off; t.table[6 * i + 2 * k + 1] = lv;
        }
    }
    if (!en.atlas.empty()) {
        const float* lut = en.srgb_lut.data();
        float mid[255];
        for (int i = 0; i < 255; i++) mid[i] = (lut[i] + lut[i + 1]) * 0.5f;
        for (const Chain& c : chains) {
            u32 w = c.w, h = c.h, off = c.off1, prev_off = 0;
            for (u32 k = 1; k < c.levels; k++) {
                const u32 sw = w, sh = h;
                if (k > 1) { prev_off = off; off += w * h; }
                w = std::max(1u, sw >> 1); h = std::max(1u, sh >> 1);
                auto src = [&](u32 x, u32 y) -> const uint8_t* {
                    if (k == 1) return en.atlas.data() + 4 * ((size_t)(c.y + y) * ATLAS_SIZE + c.x + x);
                    return t.pool.data() + 4 * ((size_t)prev_off + (size_t)y * sw + x);
                };
                for (u32 y = 0; y < h; y++) for (u32 x = 0; x < w; x++) {
                    const u32 xa = std::min(2 * x, sw - 1), xb = std::min(2 * x + 1, sw - 1), ya = std::min(2 * y, sh - 1), yb = std::min(2 * y + 1, sh - 1);
                    const uint8_t *c00 = src(xa, ya), *c10 = src(xb, ya), *c01 = src(xa, yb), *c11 = src(xb, yb);
                    uint8_t* o = t.pool.data() + 4 * ((size_t)off + (size_t)y * w + x);
                    for (int ch = 0; ch < 3; ch++) {
                        if (mutation == MUT_RAW_BYTES) { o[ch] = (uint8_t)((c00[ch] + c10[ch] + c01[ch] + c11[ch] + 2) >> 2); continue; }
                        const float s = (((lut[c00[ch]] + lut[c10[ch]]) + lut[c01[ch]]) + lut[c11[ch]]) * 0.25f;
                        u32 b = 0;
                        while (b < 255 && mid[b] < s) b++;
                        o[ch] = (uint8_t)b;
                    }
                    o[3] = (uint8_t)(((u32)c00[3] + c10[3] + c01[3] + c11[3] + 2) >> 2);
                }
            }
        }
    }
    t.built = true;
}

// texf_cone_width (st_device.cuh) over camera_ray
float cone_width(const Camera& cam, u32 px, u32 py, float t, bool primary) {
    const Ray r0 = camera_ray(cam, uv2(px, py)), r1 = camera_ray(cam, uv2(px + 1, py)), r2 = camera_ray(cam, uv2(px, py + 1));
    if (primary) return rmax_(len3((r1.origin - r0.origin) + (r1.dir - r0.dir) * t), len3((r2.origin - r0.origin) + (r2.dir - r0.dir) * t));
    return t * rmax_(len3(r1.dir - r0.dir), len3(r2.dir - r0.dir));
}
struct Foot { u32 tri; V3 dir; float w; };

float lambda_of(const Scene& sc, const Foot& f, u32 W, u32 H, u32 levels, int mutation) {
    const V4* tr = sc.triangles + 9 * (size_t)f.tri;
    const V3 p0 = xyz(tr[0]);
    const V3 c = cross3(xyz(tr[3]) - p0, xyz(tr[6]) - p0);
    const float auv = std::fabs((tr[3].w - tr[0].w) * (tr[7].w - tr[1].w) - (tr[6].w - tr[0].w) * (tr[4].w - tr[1].w));
    float cd = dot3(c, f.dir);
    if (mutation == MUT_NO_COS) cd = len3(c);
    const float q = ((((auv * (float)W) * (float)H) * (f.w * f.w)) * len3(c)) / (cd * cd);
    const float top = (float)(levels - 1);
    if (!(q > 0.0f)) return 0.0f;
    if (q == F32_INF) return top;
    return rclamp_(0.5f * log2_x(q), 0.0f, top);
}

V4 texel(const Scene& sc, const uint8_t* p) { return v4(sc.srgb_lut[p[0]], sc.srgb_lut[p[1]], sc.srgb_lut[p[2]], (float)p[3] / 255.0f); }
V4 lerp4(V4 a, V4 b, float wa, float wb) { return v4(a.x * wa + b.x * wb, a.y * wa + b.y * wb, a.z * wa + b.z * wb, a.w * wa + b.w * wb); }

V4 bilinear(const Scene& sc, const TexF& t, u32 ax, u32 ay, u32 W, u32 H, u32 off1, u32 k, float u, float v, int mutation) {
    u32 w = W, h = H, off = off1;
    for (u32 j = 1; j <= k; j++) { if (j > 1) off += w * h; w = std::max(1u, w >> 1); h = std::max(1u, h >> 1); }
    const float half = mutation == MUT_NO_HALF ? 0.0f : 0.5f;
    const float s = u * (float)w - half, tt = v * (float)h - half;
    const float sx = floorf(s), sy = floorf(tt);
    const float fx = s - sx, fy = tt - sy;
    const i32 ix = std::max(-1, std::min(f2i_sat(sx), (i32)w - 1)), iy = std::max(-1, std::min(f2i_sat(sy), (i32)h - 1));
    u32 xa = ix < 0 ? w - 1 : (u32)ix, xb = (u32)(ix + 1) >= w ? 0u : (u32)(ix + 1);
    u32 ya = iy < 0 ? h - 1 : (u32)iy, yb = (u32)(iy + 1) >= h ? 0u : (u32)(iy + 1);
    auto at_ = [&](u32 x, u32 y) -> V4 {
        if (k == 0) {
            if (mutation == MUT_CLAMP_ATLAS) {   // taps that left the image read the atlas neighbour (clamped to the atlas)
                i32 gx = (i32)ax + (x == w - 1 && ix < 0 ? -1 : (x == 0 && ix + 1 >= (i32)w ? (i32)w : (i32)x));
                i32 gy = (i32)ay + (y == h - 1 && iy < 0 ? -1 : (y == 0 && iy + 1 >= (i32)h ? (i32)h : (i32)y));
                gx = std::max(0, std::min(gx, (i32)ATLAS_SIZE - 1)); gy = std::max(0, std::min(gy, (i32)ATLAS_SIZE - 1));
                return texel(sc, sc.atlas + 4 * ((size_t)gy * ATLAS_SIZE + gx));
            }
            return texel(sc, sc.atlas + 4 * ((size_t)(ay + y) * ATLAS_SIZE + ax + x));
        }
        return texel(sc, t.pool.data() + 4 * ((size_t)off + (size_t)y * w + x));
    };
    const V4 c00 = at_(xa, ya), c10 = at_(xb, ya), c01 = at_(xa, yb), c11 = at_(xb, yb);
    const float gx = 1.0f - fx, gy = 1.0f - fy;
    return lerp4(lerp4(c00, c10, gx, fx), lerp4(c01, c11, gx, fx), gy, fy);
}

V4 sample(const Scene& sc, const TexF& t, u32 material_id, u32 slot, V4 rect, V4 mult, V2 hit_uv, const Foot& f, int mutation) {
    if (is_zero(rect) || !sc.atlas) return material_sample_atlas(sc, hit_uv, mult, rect);
    const u32 levels = std::max(t.table[6 * (size_t)material_id + 2 * slot + 1], 1u), off1 = t.table[6 * (size_t)material_id + 2 * slot];
    const u32 ax = f2u_sat(rect.x * (float)ATLAS_SIZE), ay = f2u_sat(rect.y * (float)ATLAS_SIZE);
    const u32 W = f2u_sat(rect.z * (float)ATLAS_SIZE), H = f2u_sat(rect.w * (float)ATLAS_SIZE);
    const float u = wrap_uv(hit_uv.x), v = wrap_uv(hit_uv.y);
    const float lambda = levels > 1 ? lambda_of(sc, f, W, H, levels, mutation) : 0.0f;
    const float lf = floorf(lambda);
    const u32 k0 = (u32)lf;
    const float fl = lambda - lf;
    V4 r = bilinear(sc, t, ax, ay, W, H, off1, k0, u, v, mutation);
    if (fl > 0.0f && k0 + 1 < levels) {
        const V4 r1 = bilinear(sc, t, ax, ay, W, H, off1, k0 + 1, u, v, mutation);
        r = mutation == MUT_SWAP_LEVELS ? lerp4(r, r1, fl, 1.0f - fl) : lerp4(r, r1, 1.0f - fl, fl);
    }
    return v4(mult.x * r.x, mult.y * r.y, mult.z * r.z, mult.w * r.w);
}

bool textured(const Material& m) { return !is_zero(m.base_color_texture) || !is_zero(m.emissive_texture) || !is_zero(m.metallic_roughness_texture); }

// K2 (orc_passes.hpp pass_ref_shading) with the filtered base colour and emissive
void texf_ref_shading(CamState& cs, const Scene& sc, const TexF& t, u32 seed, u32 depth, int mutation) {
    const Camera& cam = cs.curr_camera;
    V3 sun_dir = world_sun_dir(sc.world);
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
            color += throughput * atmosphere_sample(sc, sun_dir, ray.dir);
            rays[3 * idx] = v4z(); rays[3 * idx + 1] = v4z(); rays[3 * idx + 2] = v4(color, 0.0f);
            continue;
        }
        Material material = sc.materials[th.material_id];
        if (depth > 0) material_regularize(material);
        const TriangleHit again = ray_trace(ray, sc);
        const Foot ft = {again.triangle_id, ray.dir, cone_width(cam, p.x, p.y, again.distance, depth == 0)};
        Hit hit;
        hit.point = th.point + th.normal * 0.01f; hit.origin = ray.origin; hit.dir = ray.dir;
        hit.gbuffer.base_color = sample(sc, t, th.material_id, 0, material.base_color_texture, material.base_color, th.uv, ft, mutation);
        hit.gbuffer.normal = th.normal; hit.gbuffer.metallic = material.metallic;
        hit.gbuffer.emissive = xyz(sample(sc, t, th.material_id, 1, material.emissive_texture, material.emissive, th.uv, ft, mutation));
        hit.gbuffer.roughness = material.roughness;
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

void* orc_texf_create() { return new TexF(); }
void orc_texf_destroy(void* t) { delete (TexF*)t; }
void orc_texf_build(void* t, void* e, int mutation) { build(*(TexF*)t, *(Engine*)e, mutation); }
// Images::remove (st_remove_image): the rect is released, the next tick re-serialises the materials
void orc_texf_remove_image(void* e, uint64_t handle) {
    Engine* en = (Engine*)e;
    en->images.erase(std::remove_if(en->images.begin(), en->images.end(), [&](const Engine::ImageRect& r) { return r.handle == handle; }), en->images.end());
    en->dirty_images = true;
}
// st_read_scene("texture_mips")'s words; returns the word count, copies min(cap, count)
long orc_texf_read(void* tp, uint32_t* dst, long cap) {
    const TexF& t = *(const TexF*)tp;
    std::vector<u32> w = {(u32)t.texels, t.materials};
    w.insert(w.end(), t.table.begin(), t.table.end());
    const size_t head = w.size();
    w.resize(head + t.texels);
    if (t.texels) std::memcpy(w.data() + head, t.pool.data(), t.texels * 4);
    if (dst) std::memcpy(dst, w.data(), 4 * (size_t)std::min<long>(cap, (long)w.size()));
    return (long)w.size();
}
// The inputs and results of the filtered fetch at every hit the step `pass` of camera `cam`'s current frame shades (0 = K0 and 8 = K12,
// called right after that step; 22 = K2 at bounce `depth`, called before it), for the float64 restatement (tests/ref64_texfilter.py).
// PROBE_WORDS floats per dispatch thread (K0, K2: y * w + x; K12: its half grid): valid, triangle id bits, material id bits, the hit
// uv, the ray direction, the hit distance, primary (1) or secondary (0), the camera rays (o0, d0, o1, d1, o2, d2) of the pixel and of
// its right and lower neighbours, then the filtered base colour, emissive (w = 0) and metallic-roughness texel product (K0 only).
// Returns the record count.
static const int PROBE_WORDS = 40;
long orc_texf_probe(void* e, void* tp, int cam, int pass, int depth, int mutation, float* out, long cap) {
    Engine* en = (Engine*)e;
    const TexF& t = *(const TexF*)tp;
    if (!t.built) return -2;
    Engine::Cam* c = en->cameras[cam];
    CamState& cs = c->st;
    const Scene sc = en->scene();
    const Camera& camera = cs.curr_camera;
    const u32 f = c->frame;
    const int cur = (f % 2) == 1 ? 1 : 0;
    const long n = pass == 8 ? (long)full_grid_h(cs.h) * half_grid_w(cs.w) : (long)cs.h * cs.w;
    if (!out) return n;
    if (cap < n * PROBE_WORDS) return -3;
    std::memset(out, 0, sizeof(float) * (size_t)n * PROBE_WORDS);
    auto record = [&](long i, const Ray& ray, u32 tri, u32 mid, V2 uv, float dist, bool primary, UV2 px, const Material& m, bool with_mr) {
        float* r = out + i * PROBE_WORDS;
        const Foot ft = {tri, ray.dir, cone_width(camera, px.x, px.y, dist, primary)};
        r[0] = 1.0f; r[1] = u2f(tri); r[2] = u2f(mid); r[3] = uv.x; r[4] = uv.y; r[5] = ray.dir.x; r[6] = ray.dir.y; r[7] = ray.dir.z; r[8] = dist;
        r[9] = primary ? 1.0f : 0.0f;
        const Ray rs[3] = {camera_ray(camera, px), camera_ray(camera, uv2(px.x + 1, px.y)), camera_ray(camera, uv2(px.x, px.y + 1))};
        for (int k = 0; k < 3; k++) {
            float* q = r + 10 + 6 * k;
            q[0] = rs[k].origin.x; q[1] = rs[k].origin.y; q[2] = rs[k].origin.z; q[3] = rs[k].dir.x; q[4] = rs[k].dir.y; q[5] = rs[k].dir.z;
        }
        const V4 b = sample(sc, t, mid, 0, m.base_color_texture, m.base_color, uv, ft, mutation);
        const V4 em = sample(sc, t, mid, 1, m.emissive_texture, m.emissive, uv, ft, mutation);
        r[28] = b.x; r[29] = b.y; r[30] = b.z; r[31] = b.w; r[32] = em.x; r[33] = em.y; r[34] = em.z;
        if (with_mr) {
            const V4 mr = sample(sc, t, mid, 2, m.metallic_roughness_texture, v4(1.0f, m.roughness, m.metallic, 1.0f), uv, ft, mutation);
            r[36] = mr.x; r[37] = mr.y; r[38] = mr.z; r[39] = mr.w;
        }
    };
    if (pass == 0) {
        ORC_FOR_FULL_GRID(cs) {
            UV2 p = uv2(gx_, gy_);
            Ray ray = camera_ray(camera, p);
            TriangleHit th = ray_trace(ray, sc);
            if (trihit_is_some(th)) record((long)gy_ * cs.w + gx_, ray, th.triangle_id, th.material_id, th.uv, th.distance, true, p, sc.materials[th.material_id], true);
        }
        return n;
    }
    if (pass == 8) {
        const bool tracing = frame_is_gi_tracing(f);
        const int hw = half_grid_w(cs.w);
        ORC_FOR_HALF_GRID(cs) {
            UV2 gid = uv2(gx_, gy_);
            UV2 sp = tracing ? resolve_checkerboard(gid, f / 2) : resolve_checkerboard(gid, f);
            if (!camera_contains(camera, sp) || (int)gid.x >= cs.w || (int)gid.y >= cs.h) continue;
            size_t idx = camera_screen_to_idx(camera, sp);
            V3 origin;
            if (tracing) {
                Hit hit = load_hit(camera, cs.prim_gbuffer_d0[cur], cs.prim_gbuffer_d1[cur], cs.w, sp);
                if (!hit_is_some(hit)) continue;
                origin = hit.point;
            } else {
                GiReservoir res = gi_read(cs.gi_reservoirs[2].data(), idx);
                if (gi_is_empty(res)) continue;
                origin = res.sample.v1_point;
            }
            Ray ray = ray_new(origin, xyz(at(cs.gi_d0, cs.w, gid)));
            TriangleHit gh = ray_trace(ray, sc);
            if (trihit_is_some(gh)) record((long)gy_ * hw + gx_, ray, gh.triangle_id, gh.material_id, gh.uv, gh.distance, false, sp, sc.materials[gh.material_id], false);
        }
        return n;
    }
    if (pass == 22 && depth >= 0) {
        ORC_FOR_FULL_GRID(cs) {
            UV2 p = uv2(gx_, gy_);
            size_t idx = camera_screen_to_idx(camera, p);
            Ray ray;
            if (depth == 0) ray = camera_ray(camera, p);
            else {
                V4 d0 = cs.ref_rays[3 * idx], d1 = cs.ref_rays[3 * idx + 1];
                if (is_zero(d1)) continue;
                ray = ray_new(xyz(d0), xyz(d1));
            }
            TriangleHit th = trihit_unpack(cs.ref_hits[2 * idx], cs.ref_hits[2 * idx + 1]);
            if (!trihit_is_some(th)) continue;
            const TriangleHit again = ray_trace(ray, sc);
            record((long)gy_ * cs.w + gx_, ray, again.triangle_id, th.material_id, th.uv, again.distance, depth == 0, p, sc.materials[th.material_id], false);
        }
        return n;
    }
    return -1;
}
void orc_texf_srgb_lut(void* e, float* out) { const Engine* en = (const Engine*)e; for (size_t i = 0; i < en->srgb_lut.size(); i++) out[i] = en->srgb_lut[i]; }
void orc_texf_log2(const float* a, float* out, long n) { for (long i = 0; i < n; i++) out[i] = log2_x(a[i]); }
// Applies the filter to what step `pass` (the device's PassId: 0 = K0, 8 = K12) of camera `cam`'s current frame just stored, or runs
// the filtered K2 (pass 22, bounce `depth`) in place of the oracle's.
int orc_texf_apply(void* e, void* tp, int cam, int pass, int depth, int mutation) {
    Engine* en = (Engine*)e;
    const TexF& t = *(const TexF*)tp;
    if (!t.built) return -2;
    Engine::Cam* c = en->cameras[cam];
    CamState& cs = c->st;
    const Scene sc = en->scene();
    const Camera& camera = cs.curr_camera;
    const u32 f = c->frame;
    const int cur = (f % 2) == 1 ? 1 : 0;
    if (pass == 0) {
        ORC_FOR_FULL_GRID(cs) {
            UV2 p = uv2(gx_, gy_);
            Ray ray = camera_ray(camera, p);
            TriangleHit th = ray_trace(ray, sc);
            if (!trihit_is_some(th)) continue;
            const Material& m = sc.materials[th.material_id];
            if (!textured(m)) continue;
            const Foot ft = {th.triangle_id, ray.dir, cone_width(camera, p.x, p.y, th.distance, true)};
            const V4 mr = sample(sc, t, th.material_id, 2, m.metallic_roughness_texture, v4(1.0f, m.roughness, m.metallic, 1.0f), th.uv, ft, mutation);
            GBufferEntry g = gbuffer_default();
            g.base_color = sample(sc, t, th.material_id, 0, m.base_color_texture, m.base_color, th.uv, ft, mutation);
            g.emissive = xyz(sample(sc, t, th.material_id, 1, m.emissive_texture, m.emissive, th.uv, ft, mutation));
            g.normal = th.normal; g.metallic = mr.z; g.roughness = mr.y; g.reflectance = m.reflectance;
            V4 d0, d1; gbuffer_pack(g, &d0, &d1);
            at(cs.prim_gbuffer_d0[cur], cs.w, p).w = d0.w;
            at(cs.prim_gbuffer_d1[cur], cs.w, p) = d1;
        }
        return 0;
    }
    if (pass == 8) {
        const bool tracing = frame_is_gi_tracing(f);
        ORC_FOR_HALF_GRID(cs) {
            UV2 gid = uv2(gx_, gy_);
            UV2 sp = tracing ? resolve_checkerboard(gid, f / 2) : resolve_checkerboard(gid, f);
            if (!camera_contains(camera, sp)) continue;
            size_t idx = camera_screen_to_idx(camera, sp);
            V3 origin;
            if (tracing) {
                Hit hit = load_hit(camera, cs.prim_gbuffer_d0[cur], cs.prim_gbuffer_d1[cur], cs.w, sp);
                if (!hit_is_some(hit)) continue;
                origin = hit.point;
            } else {
                GiReservoir res = gi_read(cs.gi_reservoirs[2].data(), idx);
                if (gi_is_empty(res)) continue;
                origin = res.sample.v1_point;
            }
            Ray ray = ray_new(origin, xyz(at(cs.gi_d0, cs.w, gid)));
            TriangleHit gh = ray_trace(ray, sc);
            if (!trihit_is_some(gh)) continue;
            Material m = sc.materials[gh.material_id];
            if (!textured(m)) continue;
            material_regularize(m);
            const Foot ft = {gh.triangle_id, ray.dir, cone_width(camera, sp.x, sp.y, gh.distance, false)};
            GBufferEntry g = gbuffer_default();
            g.base_color = sample(sc, t, gh.material_id, 0, m.base_color_texture, m.base_color, gh.uv, ft, mutation);
            g.emissive = xyz(sample(sc, t, gh.material_id, 1, m.emissive_texture, m.emissive, gh.uv, ft, mutation));
            g.normal = gh.normal; g.metallic = m.metallic; g.roughness = m.roughness; g.reflectance = m.reflectance;
            V4 d1, d2; gbuffer_pack(g, &d1, &d2);
            at(cs.gi_d2, cs.w, gid) = d2;
        }
        return 0;
    }
    if (pass == 22 && depth >= 0 && depth < 31) {
        en->run_atmosphere();
        texf_ref_shading(cs, sc, t, dispatch_seed(en->seed_base, f, D_REF_SHADING + (u32)depth), (u32)depth, mutation);
        return 0;
    }
    return -1;
}

}  // extern "C"
