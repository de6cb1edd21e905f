// ORACLE EXTENSION — TEST INFRASTRUCTURE ONLY.  The light grid (ST_OPT_LIGHT_GRID) for the CPU oracle.
//
// The oracle in oracle/ restates the reference, which draws every light candidate uniformly from all slots, and stays exactly as it
// is.  This library is that oracle (oracle.cpp compiled unchanged into this translation unit) plus:
//   - the grid build (DESIGN.md §2 "Light grid"): the host's box, dims, cell size, margins and bands (engine.cu light_grid_header)
//     and the per-cell lists (kernels.cu k_light_grid_build), in the same f32 operations and order;
//   - grid versions of the three passes that draw light candidates, restated from orc_passes.hpp with the list in place of every
//     slot: K5 di_sampling (at hit.point), K13 gi_sampling_b (at the bounce hit's point) and K2 ref_shading (at the nudged hit point);
//   - the oracle's light_radiance for a batch of (point, normal, light) triples, for the zero check of the tests.
// oracle_lightgrid/pyoracle_lightgrid.py steps a frame pass by pass and runs the grid version of those three passes.
#include <cmath>
#include <limits>
#include "../oracle/oracle.cpp"

namespace {
using namespace orc;

const u32 K = 64, OVERFLOW_ = 0xffffffffu;
// Test-only mistakes (tests/test_light_grid.py shows that the checks catch each): 0 = the rule.
enum { MUT_NONE = 0, MUT_NO_MARGIN = 1, MUT_NO_BAND = 2, MUT_DROP_SUN = 3, MUT_GLOBAL_PDF = 4 };

struct Grid {
    float lo[3], cell[3], inv_cell[3], band[3], margin[3];
    u32 dims[3], light_count;
    std::vector<u32> counts, lists;   // cells + 1 (the outside list last)
    bool built = false;
};

bool cullable(const Light& l) {
    const float big = 0x1p60f, tiny = 0x1p-60f;
    if (f2u(l.d2.x) != 1u) return false;
    if (!(std::fabs(l.d0.x) <= big && std::fabs(l.d0.y) <= big && std::fabs(l.d0.z) <= big)) return false;
    if (!(std::isfinite(l.d1.x) && std::isfinite(l.d1.y) && std::isfinite(l.d1.z))) return false;
    return l.d1.w >= tiny && l.d1.w <= big;
}

void build(Grid& g, const std::vector<Light>& lights, u32 light_count, int n, int mutation) {
    std::memset(g.lo, 0, sizeof g.lo); std::memset(g.cell, 0, sizeof g.cell); std::memset(g.inv_cell, 0, sizeof g.inv_cell);
    std::memset(g.band, 0, sizeof g.band); std::memset(g.margin, 0, sizeof g.margin); std::memset(g.dims, 0, sizeof g.dims);
    g.light_count = light_count;
    const float inf = std::numeric_limits<float>::infinity();
    float lo[3] = {inf, inf, inf}, hi[3] = {-inf, -inf, -inf};
    bool any = false;
    for (u32 i = 0; i < light_count && i < lights.size(); i++) {
        const Light& l = lights[i];
        if (!cullable(l)) continue;
        any = true;
        const float c[3] = {l.d0.x, l.d0.y, l.d0.z}, r = l.d1.w;
        for (int a = 0; a < 3; a++) { lo[a] = std::min(lo[a], c[a] - r); hi[a] = std::max(hi[a], c[a] + r); }
    }
    if (any) {
        float ext[3], longest = 0.0f, m = 0.0f;
        for (int a = 0; a < 3; a++) { ext[a] = hi[a] - lo[a]; longest = std::max(longest, ext[a]); m = std::max(m, std::max(std::fabs(lo[a]), std::fabs(hi[a]))); }
        const float ulp = std::nextafter(m, inf) - m;
        for (int a = 0; a < 3; a++) {
            const float q = std::ceil(((float)n * ext[a]) / longest);
            const u32 d = q < 1.0f ? 1u : (q > (float)n ? (u32)n : (u32)q);
            g.dims[a] = d; g.lo[a] = lo[a];
            g.cell[a] = ext[a] / (float)d; g.inv_cell[a] = (float)d / ext[a];
            g.margin[a] = mutation == MUT_NO_MARGIN ? 0.0f : g.cell[a] * 0.015625f + 8.0f * ulp;
            g.band[a] = mutation == MUT_NO_BAND ? 0.0f : 0.0078125f + (2.0f * ulp) * g.inv_cell[a];
        }
    }
    const u32 ncell = g.dims[0] * g.dims[1] * g.dims[2];
    g.counts.assign(ncell + 1, 0u);
    g.lists.assign((size_t)(ncell + 1) * K, 0xffffffffu);
    for (u32 cell = 0; cell <= ncell; cell++) {
        const bool outside = cell == ncell;
        float bmin[3] = {0, 0, 0}, bmax[3] = {0, 0, 0};
        if (!outside) {
            const u32 idx[3] = {cell % g.dims[0], (cell / g.dims[0]) % g.dims[1], cell / (g.dims[0] * g.dims[1])};
            for (int a = 0; a < 3; a++) {
                bmin[a] = (g.lo[a] + (float)idx[a] * g.cell[a]) - g.margin[a];
                bmax[a] = (g.lo[a] + (float)(idx[a] + 1u) * g.cell[a]) + g.margin[a];
            }
        }
        u32 cnt = 0;
        for (u32 slot = 0; slot < light_count; slot++) {
            const Light& l = lights[slot];
            bool keep;
            if (mutation == MUT_DROP_SUN && slot == 0) keep = false;
            else if (!cullable(l)) keep = true;
            else if (outside) keep = false;
            else {
                const float c[3] = {l.d0.x, l.d0.y, l.d0.z};
                float d[3];
                for (int a = 0; a < 3; a++) d[a] = std::fmax(std::fmax(bmin[a] - c[a], c[a] - bmax[a]), 0.0f);
                const float d2 = (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2];
                const float thr = mutation == MUT_NO_MARGIN ? l.d1.w * l.d1.w : (l.d1.w * l.d1.w) * 1.00390625f;
                keep = !(d2 > thr);
            }
            if (!keep) continue;
            if (cnt < K) g.lists[(size_t)cell * K + cnt] = slot;
            cnt++;
        }
        g.counts[cell] = cnt > K ? OVERFLOW_ : cnt;
    }
    g.built = true;
}

// lgrid_list (st_device.cuh): ids == nullptr = every slot
struct List { const u32* ids; u32 n; };
List lookup(const Grid& g, V3 p) {
    List all = {nullptr, g.light_count};
    if (!(std::isfinite(p.x) && std::isfinite(p.y) && std::isfinite(p.z))) return all;
    const u32 ncell = g.dims[0] * g.dims[1] * g.dims[2];
    u32 cell = ncell;
    if (ncell > 0) {
        const float pc[3] = {p.x, p.y, p.z};
        u32 idx[3]; bool inside = true;
        for (int a = 0; a < 3; a++) {
            const float t = (pc[a] - g.lo[a]) * g.inv_cell[a];
            if (!(t >= -g.band[a]) || !(t < (float)g.dims[a] + g.band[a])) inside = false;
            idx[a] = (u32)(int)std::floor(std::fmin(std::fmax(t, 0.0f), (float)(g.dims[a] - 1u)));
        }
        if (inside) cell = (idx[2] * g.dims[1] + idx[1]) * g.dims[0] + idx[0];
    }
    const u32 c = g.counts[cell];
    if (c == OVERFLOW_) return all;
    return List{g.lists.data() + (size_t)cell * K, c};
}
u32 pick(const List& l, u32 r) { return l.ids ? l.ids[r] : r; }

// ephemeral_build (orc_gpu.hpp) over a list
EphemeralReservoir ephemeral_build_list(WhiteNoise& wn, const Scene& sc, const Hit& hit, const List& list) {
    EphemeralReservoir res; res.sample.light_id = 0; res.sample.light_rad = light_radiance_default(); res.m = 0; res.w = 0;
    float res_pdf = 0.0f;
    u32 lc = list.n;
    u32 max_samples = lc < 16 ? lc : 16;
    float sample_ipdf = (float)lc;
    for (u32 nth = 0; nth < max_samples; nth++) {
        EphemeralSample s;
        s.light_id = pick(list, wnoise_sample_int(wn) % lc);
        s.light_rad = light_radiance(sc.lights[s.light_id], hit);
        float sample_pdf = perc_luma(s.light_rad.radiance);
        if (res.update(wn, s, sample_pdf * sample_ipdf)) res_pdf = sample_pdf;
    }
    res.norm_avg(res_pdf);
    return res;
}

// K5 (orc_passes.hpp pass_di_sampling) with the list of hit.point
void grid_di_sampling(CamState& cs, const Scene& sc, const Grid& g, bool alternate, u32 seed, u32 frame) {
    int cur = alternate ? 1 : 0;
    const Camera& cam = cs.curr_camera;
    ORC_FOR_FULL_GRID(cs) {
        UV2 p = uv2(gx_, gy_);
        size_t idx = camera_screen_to_idx(cam, p);
        WhiteNoise wn = wnoise_new(seed, p);
        Hit hit = load_hit(cam, cs.prim_gbuffer_d0[cur], cs.prim_gbuffer_d1[cur], cs.w, p);
        if (!hit_is_some(hit)) continue;
        EphemeralReservoir res = ephemeral_build_list(wn, sc, hit, lookup(g, hit.point));
        DiReservoir out = di_default();
        if (res.m > 0.0f) {
            V4 bn = bnoise_texel(sc.blue_noise, p, frame);
            Ray ray = light_ray_bnoise(sc.lights[res.sample.light_id], v2(bn.x, bn.y), hit.point);
            bool is_occluded = ray_intersect(ray, sc);
            if (is_occluded) res.w = 0.0f;
            out.sample.pdf = 0.0f; out.sample.confidence = 0.0f; out.sample.light_id = res.sample.light_id;
            out.sample.light_point = ray.origin; out.sample.is_occluded = is_occluded;
            out.m = 1.0f; out.w = res.w;
        }
        di_write(out, cs.di_reservoirs[1].data(), idx);
    }
}

// K13 (orc_passes.hpp pass_gi_sampling_b) with the list of the bounce hit's point; the sky-or-light draw keeps the global count
void grid_gi_sampling_b(CamState& cs, const Scene& sc, const Grid& g, bool alternate, u32 seed, u32 frame) {
    int cur = alternate ? 1 : 0;
    const Camera& cam = cs.curr_camera;
    bool tracing = frame_is_gi_tracing(frame);
    V3 sun_dir = world_sun_dir(sc.world);
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
        if (!hit_is_some(gi_hit)) {
            light_id = SKY; light_pdf = 1.0f; light_rad = atmosphere_sample(sc, sun_dir, gi_hit.dir);
        } else {
            float atmosphere_pdf = (sc.world.sun_altitude <= -1.0f) ? 0.0f : 0.25f;
            if (sc.world.light_count == 0 || wnoise_sample(wn) < atmosphere_pdf) {
                light_id = SKY; light_pdf = atmosphere_pdf;
                light_dir = wnoise_sample_hemisphere(wn, gi_hit.gbuffer.normal);
                light_rad = atmosphere_sample(sc, sun_dir, light_dir) * dot(gi_hit.gbuffer.normal, light_dir);
            } else {
                EphemeralReservoir res = ephemeral_build_list(wn, sc, gi_hit, lookup(g, gi_hit.point));
                if (res.w > 0.0f) {
                    light_id = res.sample.light_id;
                    light_pdf = (1.0f / res.w) * (1.0f - atmosphere_pdf);
                    light_rad = res.sample.light_rad.radiance * (v3s(1.0f) + res.sample.light_rad.spec_brdf);
                } else { light_id = 0; light_pdf = 1.0f; light_rad = v3s(0); }
            }
        }
        V3 radiance;
        if (light_pdf > 0.0f) {
            float light_vis;
            if (hit_is_some(gi_hit)) {
                Ray ray = (light_id == SKY) ? ray_new(gi_hit.point, light_dir) : light_ray_wnoise(sc.lights[light_id], wn, gi_hit.point);
                light_vis = ray_intersect(ray, sc) ? 0.0f : 1.0f;
            } else light_vis = 1.0f;
            radiance = light_rad * light_vis / light_pdf;
        } else radiance = v3s(0);
        if (hit_is_some(gi_hit)) {
            radiance *= xyz(gi_hit.gbuffer.base_color) / PI;
            radiance += gi_hit.gbuffer.emissive;
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

// K2 (orc_passes.hpp pass_ref_shading) with the list of the nudged hit point; depth 255 (accumulation) draws no light
void grid_ref_shading(CamState& cs, const Scene& sc, const Grid& g, u32 seed, u32 depth, int mutation) {
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
        Hit hit;
        hit.point = th.point + th.normal * 0.01f; hit.origin = ray.origin; hit.dir = ray.dir;
        hit.gbuffer.base_color = material_base_color(sc, material, th.uv); hit.gbuffer.normal = th.normal; hit.gbuffer.metallic = material.metallic;
        hit.gbuffer.emissive = material_emissive(sc, material, th.uv); hit.gbuffer.roughness = material.roughness;
        hit.gbuffer.reflectance = material.reflectance; hit.gbuffer.depth = 0.0f;
        color += throughput * hit.gbuffer.emissive;
        const List list = lookup(g, hit.point);
        if (list.n > 0) {
            u32 light_id = pick(list, wnoise_sample_int(wn) % list.n);
            float light_pdf = 1.0f / (float)(mutation == MUT_GLOBAL_PDF ? sc.world.light_count : list.n);
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

void* orc_lgrid_create() { return new Grid(); }
void orc_lgrid_destroy(void* g) { delete (Grid*)g; }
// Builds the grid of `n` cells along the longest axis over the lights the engine's frames see (gpu_lights, world.light_count).
void orc_lgrid_build(void* g, void* e, int n, int mutation) {
    Engine* en = (Engine*)e;
    build(*(Grid*)g, en->gpu_lights, en->world.light_count, n, mutation);
}
// st_read_scene("light_grid")'s words (include/strolle_b200.h); returns the word count, copies min(cap, count)
long orc_lgrid_read(void* gp, uint32_t* dst, long cap) {
    const Grid& g = *(const Grid*)gp;
    const u32 ncell = g.dims[0] * g.dims[1] * g.dims[2];
    std::vector<u32> w = {g.dims[0], g.dims[1], g.dims[2], K, g.light_count, ncell};
    for (const float* v : {g.lo, g.cell, g.inv_cell, g.band, g.margin}) for (int a = 0; a < 3; a++) w.push_back(f2u(v[a]));
    w.insert(w.end(), g.counts.begin(), g.counts.end());
    w.insert(w.end(), g.lists.begin(), g.lists.end());
    if (dst) std::memcpy(dst, w.data(), 4 * (size_t)std::min<long>(cap, (long)w.size()));
    return (long)w.size();
}
// The list each point samples: out_n = its length, or 0xffffffff for every slot; out_ids = K words per point
void orc_lgrid_point_lists(void* gp, const float* pts, long n, uint32_t* out_n, uint32_t* out_ids) {
    const Grid& g = *(const Grid*)gp;
    for (long i = 0; i < n; i++) {
        List l = lookup(g, v3(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]));
        out_n[i] = l.ids ? l.n : OVERFLOW_;
        for (u32 k = 0; k < K; k++) out_ids[(size_t)i * K + k] = (l.ids && k < l.n) ? l.ids[k] : OVERFLOW_;
    }
}
// light_radiance(lights[id], hit).radiance for hits at `pts` with shading normal `nrm` (dielectric, roughness 1, white)
void orc_lgrid_radiance(void* e, const float* pts, const float* nrm, const uint32_t* ids, long n, float* out3) {
    Engine* en = (Engine*)e;
    const Scene sc = en->scene();
    for (long i = 0; i < n; i++) {
        Hit h = hit_default();
        h.point = v3(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]);
        h.gbuffer.normal = v3(nrm[3 * i], nrm[3 * i + 1], nrm[3 * i + 2]);
        h.gbuffer.base_color = v4(1, 1, 1, 1); h.gbuffer.roughness = 1.0f; h.gbuffer.reflectance = 0.5f;
        h.dir = -h.gbuffer.normal; h.origin = h.point + h.gbuffer.normal;
        V3 r = light_radiance(sc.lights[ids[i]], h).radiance;
        out3[3 * i] = r.x; out3[3 * i + 1] = r.y; out3[3 * i + 2] = r.z;
    }
}
// Runs the grid version of step `pass` (the device's PassId: 1 = K5, 9 = K13, 22 = K2 at bounce `depth`) of camera `cam`'s current
// frame in place of the oracle's.  Call it where render_range would run that step.
int orc_lgrid_step(void* e, void* gp, int cam, int pass, int depth, int mutation) {
    Engine* en = (Engine*)e;
    const Grid& g = *(const Grid*)gp;
    if (!g.built) return -2;
    en->run_atmosphere();
    Engine::Cam* c = en->cameras[cam];
    const Scene sc = en->scene();
    const u32 f = c->frame;
    const bool alt = (f % 2) == 1;
    if (pass == D_DI_SAMPLING) { grid_di_sampling(c->st, sc, g, alt, dispatch_seed(en->seed_base, f, D_DI_SAMPLING), f); return 0; }
    if (pass == D_GI_SAMPLING_B) { grid_gi_sampling_b(c->st, sc, g, alt, dispatch_seed(en->seed_base, f, D_GI_SAMPLING_B), f); return 0; }
    if (pass == 22 && depth >= 0 && depth < 31) { grid_ref_shading(c->st, sc, g, dispatch_seed(en->seed_base, f, D_REF_SHADING + (u32)depth), (u32)depth, mutation); return 0; }
    return -1;
}

}  // extern "C"
