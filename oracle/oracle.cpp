// ORACLE — TEST INFRASTRUCTURE ONLY (see orc_math.hpp header).
// C ABI over the oracle for ctypes (tests/, smoke(), bench.py cpu_baseline).
#include <cstdio>
#include <cstring>
#include "orc_host.hpp"

using namespace orc;

static M4 m4_from(const float* p) { M4 m; std::memcpy(&m, p, 64); return m; }
static HostCamera host_camera(int mode, int denoise, int ref_depth, int w, int h, const float* transform16, const float* projection16) {
    HostCamera hc; hc.mode = mode; hc.denoise = denoise != 0; hc.ref_depth = (u32)ref_depth; hc.w = (u32)w; hc.h = (u32)h;
    hc.transform = m4_from(transform16); hc.projection = m4_from(projection16); return hc;
}

extern "C" {

void* orc_engine_create() { return new Engine(); }
void orc_engine_destroy(void* e) { delete (Engine*)e; }
void orc_set_blue_noise(void* e, const uint8_t* rgba) { ((Engine*)e)->blue_noise.assign(rgba, rgba + 256 * 256 * 4); }
void orc_set_seed_base(void* e, uint32_t base) { ((Engine*)e)->seed_base = base; }
uint32_t orc_frame(void* e) { return ((Engine*)e)->frame; }

// tris: per triangle 36 floats = positions[3][3], normals[3][3], uvs[3][2], tangents[3][4]
void orc_insert_mesh(void* e, uint64_t handle, const float* tris, int n) {
    std::vector<MeshTriangle> v((size_t)n);
    for (int i = 0; i < n; i++) {
        const float* p = tris + 36 * (size_t)i;
        for (int k = 0; k < 3; k++) {
            v[i].positions[k] = v3(p[3 * k], p[3 * k + 1], p[3 * k + 2]);
            v[i].normals[k] = v3(p[9 + 3 * k], p[9 + 3 * k + 1], p[9 + 3 * k + 2]);
            v[i].uvs[k] = v2(p[18 + 2 * k], p[18 + 2 * k + 1]);
            v[i].tangents[k] = v4(p[24 + 4 * k], p[24 + 4 * k + 1], p[24 + 4 * k + 2], p[24 + 4 * k + 3]);
        }
    }
    ((Engine*)e)->insert_mesh(handle, v);
}
// p: base_color[4], emissive[4], perceptual_roughness, metallic, reflectance, ior
void orc_insert_material(void* e, uint64_t handle, const float* p, int alpha_blend) {
    HostMaterial m; m.base_color = v4(p[0], p[1], p[2], p[3]); m.emissive = v4(p[4], p[5], p[6], p[7]);
    m.perceptual_roughness = p[8]; m.metallic = p[9]; m.reflectance = p[10]; m.ior = p[11]; m.alpha_blend = alpha_blend != 0;
    ((Engine*)e)->insert_material(handle, m);
}
int orc_insert_image(void* e, uint64_t handle, const uint8_t* rgba, int w, int h) { return ((Engine*)e)->insert_image(handle, rgba, (u32)w, (u32)h) ? 0 : -1; }
// tex[i] for i in base_color, emissive, metallic_roughness, normal_map; mask bit i = texture present
void orc_set_material_textures(void* e, uint64_t handle, const uint64_t* tex, uint32_t mask) {
    Engine* en = (Engine*)e;
    for (auto& p : en->material_index) if (p.first == handle) {
        for (int i = 0; i < 4; i++) { en->materials[p.second].tex[i] = tex[i]; en->materials[p.second].has_tex[i] = (mask >> i) & 1u; }
        en->dirty_materials = true;
    }
}
// affine12: matrix3 columns x,y,z then translation
void orc_insert_instance(void* e, uint64_t handle, uint64_t mesh, uint64_t material, const float* a) {
    Affine xf; xf.x = v3(a[0], a[1], a[2]); xf.y = v3(a[3], a[4], a[5]); xf.z = v3(a[6], a[7], a[8]); xf.t = v3(a[9], a[10], a[11]);
    ((Engine*)e)->insert_instance(handle, mesh, material, xf);
}
void orc_remove_instance(void* e, uint64_t handle) { ((Engine*)e)->remove_instance(handle); }
// p: position[3], radius, color[3], range, direction[3], angle ; type 1 = point, 2 = spot
void orc_insert_light(void* e, uint64_t handle, int type, const float* p) {
    HostLight l; l.type = type; l.position = v3(p[0], p[1], p[2]); l.radius = p[3]; l.color = v3(p[4], p[5], p[6]); l.range = p[7];
    l.direction = v3(p[8], p[9], p[10]); l.angle = p[11];
    ((Engine*)e)->insert_light(handle, l);
}
void orc_remove_light(void* e, uint64_t handle) { ((Engine*)e)->remove_light(handle); }
void orc_update_sun(void* e, float azimuth, float altitude) { ((Engine*)e)->update_sun(azimuth, altitude); }
int orc_create_camera(void* e, int mode, int denoise, int ref_depth, int w, int h, const float* transform16, const float* projection16) {
    return ((Engine*)e)->create_camera(host_camera(mode, denoise, ref_depth, w, h, transform16, projection16));
}
void orc_update_camera(void* e, int cam, int mode, int denoise, int ref_depth, int w, int h, const float* transform16, const float* projection16) {
    ((Engine*)e)->update_camera(cam, host_camera(mode, denoise, ref_depth, w, h, transform16, projection16));
}
void orc_tick(void* e) { ((Engine*)e)->tick(); }
void orc_render_camera(void* e, int cam) { ((Engine*)e)->render_camera(cam); }
void orc_render_range(void* e, int cam, int first, int last) { ((Engine*)e)->render_range(cam, first, last); }
// pass ids of this frame's steps (the device's PassId values); returns the step count, copies min(cap, count)
int orc_frame_schedule(void* e, int cam, int* ids, int cap) {
    Engine* en = (Engine*)e;
    en->run_atmosphere();
    std::vector<Engine::Step> steps = en->schedule(cam);
    for (int i = 0; i < cap && i < (int)steps.size(); i++) ids[i] = steps[i].pass;
    return (int)steps.size();
}

// returns number of floats available; copies min(cap, n)
long orc_read_buffer(void* e, int cam, const char* name, float* dst, long cap) {
    Engine* en = (Engine*)e;
    Buf* b = en->cameras[cam]->st.by_name(name);
    if (!b) {
        if (std::strcmp(name, "curr_camera") == 0 || std::strcmp(name, "prev_camera") == 0) {
            const Camera& c = std::strcmp(name, "curr_camera") == 0 ? en->cameras[cam]->st.curr_camera : en->cameras[cam]->st.prev_camera;
            long n = 40; if (dst) std::memcpy(dst, &c, sizeof(float) * (size_t)(cap < n ? cap : n)); return n;
        }
        return -1;
    }
    long n = (long)b->size() * 4;
    if (dst) std::memcpy(dst, b->data(), sizeof(float) * (size_t)(cap < n ? cap : n));
    return n;
}
long orc_read_scene(void* e, const char* name, float* dst, long cap) {
    Engine* en = (Engine*)e;
    const void* src = nullptr; long n = 0;
    std::string s(name);
    if (s == "triangles") { src = en->gpu_triangles.data(); n = (long)en->gpu_triangles.size() * 4; }
    else if (s == "bvh") { src = en->gpu_bvh.data(); n = (long)en->gpu_bvh.size() * 4; }
    else if (s == "materials") { src = en->gpu_materials.data(); n = (long)en->gpu_materials.size() * 28; }
    else if (s == "lights") { src = en->gpu_lights.data(); n = (long)en->gpu_lights.size() * 28; }
    else if (s == "world") { src = &en->world; n = 4; }
    else if (s == "transmittance_lut") { en->run_atmosphere(); src = en->luts.transmittance.data(); n = (long)en->luts.transmittance.size() * 4; }
    else if (s == "scattering_lut") { en->run_atmosphere(); src = en->luts.scattering.data(); n = (long)en->luts.scattering.size() * 4; }
    else if (s == "sky_lut") { en->run_atmosphere(); src = en->luts.sky.data(); n = (long)en->luts.sky.size() * 4; }
    else return -1;
    if (dst) std::memcpy(dst, src, sizeof(float) * (size_t)(cap < n ? cap : n));
    return n;
}
int orc_bvh_depth(void* e) { return ((Engine*)e)->bvh_depth; }

// Ray-stream hooks (the Mrays/s micro-benchmark shape, K1/K8/K16).
// rays: 8 floats per ray (origin xyz, len, dir xyz, pad).
// closest: out 12 floats per ray = packed hit d0,d1 (hit.rs:112-120), then (distance, bits triangle_id, bits material_id, used_memory as f32)
void orc_trace_closest(void* e, const float* rays, long n, float* out) {
    Engine* en = (Engine*)e; Scene sc = en->scene();
    _Pragma("omp parallel for schedule(dynamic, 256)")
    for (long i = 0; i < n; i++) {
        const float* r = rays + 8 * i;
        Ray ray = ray_new(v3(r[0], r[1], r[2]), v3(r[4], r[5], r[6]));
        size_t used = 0;
        TriangleHit h = ray_trace(ray, sc, &used);
        V4 d0, d1; trihit_pack(h, &d0, &d1);
        float* o = out + 12 * i;
        std::memcpy(o, &d0, 16); std::memcpy(o + 4, &d1, 16);
        o[8] = h.distance; o[9] = u2f(h.triangle_id); o[10] = u2f(h.material_id); o[11] = (float)used;
    }
}
void orc_trace_any(void* e, const float* rays, long n, uint32_t* out) {
    Engine* en = (Engine*)e; Scene sc = en->scene();
    _Pragma("omp parallel for schedule(dynamic, 256)")
    for (long i = 0; i < n; i++) {
        const float* r = rays + 8 * i;
        Ray ray = ray_with_len(ray_new(v3(r[0], r[1], r[2]), v3(r[4], r[5], r[6])), r[3]);
        out[i] = ray_intersect(ray, sc) ? 1u : 0u;
    }
}
// brute force over every triangle (self-check of the traversal, SURVEY §8c)
void orc_trace_brute(void* e, const float* rays, long n, float* out_dist, uint32_t* out_tri) {
    Engine* en = (Engine*)e; Scene sc = en->scene();
    long ntri = (long)en->gpu_triangles.size() / 9;
    _Pragma("omp parallel for schedule(dynamic, 256)")
    for (long i = 0; i < n; i++) {
        const float* r = rays + 8 * i;
        Ray ray = ray_new(v3(r[0], r[1], r[2]), v3(r[4], r[5], r[6]));
        TriangleHit h = trihit_none();
        for (long t = 0; t < ntri; t++) if (triangle_hit(sc.triangles + 9 * t, ray, &h)) h.triangle_id = (u32)t;
        out_dist[i] = h.distance; out_tri[i] = h.triangle_id;
    }
}

// elementary-function hooks: op 0 sin,1 cos,2 acos,3 atan2(a,b),4 exp,5 pow(a,b),6 glam acos_approx,7 round_f16
void orc_math(int op, const float* a, const float* b, float* out, long n) {
    for (long i = 0; i < n; i++) {
        switch (op) {
            case 0: out[i] = sin_(a[i]); break;
            case 1: out[i] = cos_(a[i]); break;
            case 2: out[i] = acos_(a[i]); break;
            case 3: out[i] = atan2_(a[i], b[i]); break;
            case 4: out[i] = exp_(a[i]); break;
            case 5: out[i] = pow_(a[i], b[i]); break;
            case 6: out[i] = acos_approx(a[i]); break;
            case 7: out[i] = round_f16(a[i]); break;
            default: out[i] = 0.0f;
        }
    }
}

// --- hooks for the six reference unit tests (SURVEY §4) ---------------------
void orc_gbuffer_pack(const float* g /*base_color4, normal3, metallic, emissive3, roughness, reflectance, depth*/, float* out8) {
    GBufferEntry e; e.base_color = v4(g[0], g[1], g[2], g[3]); e.normal = v3(g[4], g[5], g[6]); e.metallic = g[7]; e.emissive = v3(g[8], g[9], g[10]);
    e.roughness = g[11]; e.reflectance = g[12]; e.depth = g[13];
    V4 d0, d1; gbuffer_pack(e, &d0, &d1); std::memcpy(out8, &d0, 16); std::memcpy(out8 + 4, &d1, 16);
}
void orc_gbuffer_unpack(const float* in8, float* g) {
    V4 d0, d1; std::memcpy(&d0, in8, 16); std::memcpy(&d1, in8 + 4, 16);
    GBufferEntry e = gbuffer_unpack(d0, d1);
    g[0] = e.base_color.x; g[1] = e.base_color.y; g[2] = e.base_color.z; g[3] = e.base_color.w; g[4] = e.normal.x; g[5] = e.normal.y; g[6] = e.normal.z;
    g[7] = e.metallic; g[8] = e.emissive.x; g[9] = e.emissive.y; g[10] = e.emissive.z; g[11] = e.roughness; g[12] = e.reflectance; g[13] = e.depth;
}
void orc_camera_contain(float sw, float sh, int x, int y, uint32_t* out2) {
    Camera c; std::memset(&c, 0, sizeof c); c.screen = v4(sw, sh, 0, 0);
    UV2 r = camera_contain(c, iv2(x, y)); out2[0] = r.x; out2[1] = r.y;
}
// in: m, w, pdf, confidence, light_id(bits), light_point3, is_occluded ; writes slot `idx` of buf then reads it back
void orc_di_reservoir_roundtrip(float* buf, long idx, const float* in9, float* out9) {
    DiReservoir r; r.m = in9[0]; r.w = in9[1]; r.sample.pdf = in9[2]; r.sample.confidence = in9[3]; r.sample.light_id = f2u(in9[4]);
    r.sample.light_point = v3(in9[5], in9[6], in9[7]); r.sample.is_occluded = in9[8] != 0.0f;
    di_write(r, (V4*)buf, (size_t)idx);
    DiReservoir q = di_read((const V4*)buf, (size_t)idx);
    out9[0] = q.m; out9[1] = q.w; out9[2] = q.sample.pdf; out9[3] = q.sample.confidence; out9[4] = u2f(q.sample.light_id);
    out9[5] = q.sample.light_point.x; out9[6] = q.sample.light_point.y; out9[7] = q.sample.light_point.z; out9[8] = q.sample.is_occluded ? 1.0f : 0.0f;
}
void orc_reprojection_roundtrip(const float* in3, uint32_t validity, float* out3, uint32_t* out_validity) {
    Reprojection r = {in3[0], in3[1], in3[2], validity};
    Reprojection q = reprojection_deserialize(reprojection_serialize(r));
    out3[0] = q.prev_x; out3[1] = q.prev_y; out3[2] = q.confidence; *out_validity = q.validity;
}
uint32_t orc_u32_bytes_roundtrip(uint32_t v) { return from_bytes(v & 0xff, (v >> 8) & 0xff, (v >> 16) & 0xff, (v >> 24) & 0xff); }
// allocator script: ops[i] = {0 give(a,b) | 1 take(a)}; out[i] = {found, start, end}
void orc_allocator_script(const long* ops, int n, long* out) {
    Allocator al;
    for (int i = 0; i < n; i++) {
        long op = ops[3 * i], a = ops[3 * i + 1], b = ops[3 * i + 2];
        out[3 * i] = out[3 * i + 1] = out[3 * i + 2] = 0;
        if (op == 0) al.give((size_t)a, (size_t)b);
        else { size_t s, e; if (al.take((size_t)a, &s, &e)) { out[3 * i] = 1; out[3 * i + 1] = (long)s; out[3 * i + 2] = (long)e; } }
    }
}
// BVH builder on its own (strolle/src/bvh/builder.rs + serializer.rs): prims = n x 11 floats (triangle id bits, material id bits,
// centre, bounds min, bounds max); the handle keeps the previous tree for subtree reuse (builder.rs:245-359).
void* orc_bvh_builder_create() { return new BvhBuilder(); }
void orc_bvh_builder_destroy(void* b) { delete (BvhBuilder*)b; }
long orc_bvh_builder_build(void* bp, const float* prims11, long n, int reuse, float* out, long cap_floats, uint32_t* reused, int* depth) {
    BvhBuilder* b = (BvhBuilder*)bp;
    std::vector<BvhPrimitive> all((size_t)n);
    u32 max_mat = 0;
    for (long i = 0; i < n; i++) {
        const float* f = prims11 + 11 * i;
        BvhPrimitive& p = all[(size_t)i];
        p.triangle_id = f2u(f[0]); p.material_id = f2u(f[1]); p.center = v3(f[2], f[3], f[4]);
        p.bounds = BBox(); p.bounds.mn = v3(f[5], f[6], f[7]); p.bounds.mx = v3(f[8], f[9], f[10]);
        max_mat = std::max(max_mat, p.material_id);
    }
    b->reuse = reuse != 0;
    b->run(all);
    for (const BvhPrimitive& p : b->prims) max_mat = std::max(max_mat, p.material_id);
    std::vector<uint8_t> alpha((size_t)max_mat + 1, 0);
    std::vector<V4> buf; int d = 0;
    b->serialize(buf, alpha, 0, 1, &d);
    if (reused) *reused = b->reused_subtrees;
    if (depth) *depth = d;
    long nf = (long)buf.size() * 4;
    if (out && cap_floats >= nf) std::memcpy(out, buf.data(), (size_t)nf * 4);
    return nf;
}
void orc_set_bvh_reuse(void* e, int reuse) { ((Engine*)e)->bvh.reuse = reuse != 0; }
uint32_t orc_bvh_reused(void* e) { return ((Engine*)e)->bvh.reused_subtrees; }

unsigned long long orc_ray_count(int reset) {
    unsigned long long t = 0;
    for (int i = 0; i < 256; i++) { t += g_ray_counters[i].n; if (reset) g_ray_counters[i].n = 0; }
    return t;
}
void orc_set_threads(int n) {
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
#endif
}
int orc_get_threads() {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}
int orc_is_libm() {
#ifdef ORC_LIBM
    return 1;
#else
    return 0;
#endif
}

}  // extern "C"
