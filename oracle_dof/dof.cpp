// ORACLE EXTENSION — TEST INFRASTRUCTURE ONLY.  Depth of field (ST_OPT_DEPTH_OF_FIELD) for the CPU oracle.
//
// This library is the oracle (oracle/oracle.cpp compiled unchanged into this translation unit, for its camera rays) plus the rule of
// DESIGN.md §2 "Depth of field" in the oracle's own arithmetic:
//   - orc_dof_taps: the gather's tap table;
//   - orc_dof_consts: the lens constants of a frame, from the settings, the camera transform and projection;
//   - orc_dof_run: the "depth_of_field" words and the defocused frame of a frame's `output` and primary hit distances;
//   - orc_dof_lens / orc_dof_lens_rays: Reference mode's lens constants and thin-lens primary rays;
//   - orc_dof_render_reference: a Reference-mode frame of an oracle engine with K1 / K2's depth-0 rays leaving the thin lens.
// oracle_dof/pyoracle_dof.py calls these where the device defocuses.
#include "../oracle/oracle.cpp"

namespace {
using namespace orc;

// Test-only mistakes (tests/test_depth_of_field.py shows that the float64 bound catches each): 0 = the rule.
enum { DM_NONE = 0, DM_SIGN = 1, DM_RAY_DISTANCE = 2, DM_NO_BACKGROUND_LIMIT = 3, DM_NO_DENSITY = 4, DM_NO_DILATION = 5, DM_TRUNCATED = 6,
       DM_SKY_IN_FOCUS = 7, DM_NAN_KEPT = 8, DM_LENS_SHADING_STREAM = 9 };
const u32 kLensDispatch = 27;   // K_LENS (engine.cu)
const int kTile = 16, kMaxRadius = 32, kTaps = 81, kHeader = 16;

struct Tap { int dx, dy; float d; };

long round_half_away(double v) { return v < 0.0 ? -(long)std::floor(-v + 0.5) : (long)std::floor(v + 0.5); }

std::vector<Tap> taps_of(int mut) {
    std::vector<Tap> t;
    for (int rho = 1; rho <= kMaxRadius; rho++) {
        t.push_back(Tap{0, 0, 0.0f});
        for (int j = 1; j <= 4; j++)
            for (int i = 0; i < 8 * j; i++) {
                const double a = 2.0 * M_PI * i / (8 * j), rad = rho * j / 4.0;
                const double vx = rad * std::cos(a), vy = rad * std::sin(a);
                const long dx = mut == DM_TRUNCATED ? (long)vx : round_half_away(vx), dy = mut == DM_TRUNCATED ? (long)vy : round_half_away(vy);
                t.push_back(Tap{(int)dx, (int)dy, (float)std::sqrt((double)(dx * dx + dy * dy))});
            }
    }
    return t;
}

// consts: {f, A, k, F, R, fwd.x, fwd.y, fwd.z}; returns whether the frame is defocused
int consts_of(const float* lens, const float* transform, const float* projection, int H, float* out) {
    const double f = 0.5 * (double)lens[2] * (double)projection[5], A = f / (double)lens[1], F = (double)lens[0];
    const bool active = F > f;
    const double k = active ? A * f / (F - f) * (double)H / (double)lens[2] / 2.0 : 0.0;
    const double fx = -(double)transform[8], fy = -(double)transform[9], fz = -(double)transform[10];
    const double n = std::sqrt(fx * fx + fy * fy + fz * fz);
    out[0] = (float)f; out[1] = (float)A; out[2] = (float)k; out[3] = lens[0]; out[4] = lens[3];
    out[5] = (float)(fx / n); out[6] = (float)(fy / n); out[7] = (float)(fz / n);
    return active ? 1 : 0;
}

// Reference mode's lens: {h, F, right.xyz, up.xyz, fwd.xyz}; returns whether the rays leave a lens (F > f)
int lens_of(const float* lens, const float* transform, const float* projection, float* out) {
    const double f = 0.5 * (double)lens[2] * (double)projection[5], A = f / (double)lens[1];
    out[0] = (float)(A / 2.0); out[1] = lens[0];
    for (int k = 0; k < 3; k++) {
        const double sg = k == 2 ? -1.0 : 1.0;
        const double x = sg * transform[4 * k], y = sg * transform[4 * k + 1], z = sg * transform[4 * k + 2], n = std::sqrt(x * x + y * y + z * z);
        out[2 + 3 * k] = (float)(x / n); out[3 + 3 * k] = (float)(y / n); out[4 + 3 * k] = (float)(z / n);
    }
    return (double)lens[0] > f ? 1 : 0;
}
// The thin-lens ray of pixel p: a uniform point of the unit disc by rejection (at most 16 pairs of the lens stream, else the centre),
// the origin o + (right (h u.x) + up (h u.y)), aimed at the pinhole ray's point at view depth F
Ray lens_ray(const Camera& cam, const float* L, u32 seed, UV2 p) {
    const Ray pin = camera_ray(cam, p);
    WhiteNoise wn = wnoise_new(seed, p);
    float a = 0.0f, b = 0.0f;
    for (int i = 0; i < 16; i++) {
        const float u = wnoise_sample(wn) * 2.0f - 1.0f, v = wnoise_sample(wn) * 2.0f - 1.0f;
        if (u * u + v * v <= 1.0f) { a = u; b = v; break; }
    }
    const float ha = L[0] * a, hb = L[0] * b;
    const V3 o = pin.origin + (v3(L[2], L[3], L[4]) * ha + v3(L[5], L[6], L[7]) * hb);
    const float sc = L[1] / ((pin.dir.x * L[8] + pin.dir.y * L[9]) + pin.dir.z * L[10]);
    const V3 pf = pin.origin + pin.dir * sc;
    return ray_new(o, normalize(pf - o));
}
// K1 and K2 (oracle/orc_passes.hpp pass_ref_tracing, pass_ref_shading) with the depth-0 ray of lens_ray
void ref_tracing_lens(CamState& cs, const Scene& sc, u32 depth, const float* L, u32 lseed) {
    const Camera& cam = cs.curr_camera;
    ORC_FOR_FULL_GRID(cs) {
        UV2 p = uv2(gx_, gy_);
        size_t idx = camera_screen_to_idx(cam, p);
        Ray ray;
        if (depth == 0) ray = lens_ray(cam, L, lseed, p);
        else {
            V4 d0 = cs.ref_rays[3 * idx], d1 = cs.ref_rays[3 * idx + 1];
            if (is_zero(d1)) continue;
            ray = ray_new(xyz(d0), xyz(d1));
        }
        TriangleHit h = ray_trace(ray, sc);
        trihit_pack(h, &cs.ref_hits[2 * idx], &cs.ref_hits[2 * idx + 1]);
    }
}
void ref_shading_lens(CamState& cs, const Scene& sc, u32 seed, u32 depth, const float* L, u32 lseed) {
    const Camera& cam = cs.curr_camera;
    V3 sun_dir = world_sun_dir(sc.world);
    ORC_FOR_FULL_GRID(cs) {
        UV2 p = uv2(gx_, gy_);
        size_t idx = camera_screen_to_idx(cam, p);
        WhiteNoise wn = wnoise_new(seed, p);
        V4* rays = cs.ref_rays.data();
        Ray ray; V3 color, throughput;
        if (depth == 0) { ray = lens_ray(cam, L, lseed, p); color = v3s(0); throughput = v3s(1.0f); }
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

float finite_or_0(float v, int mut) { return (mut == DM_NAN_KEPT || std::fabs(v) < std::numeric_limits<float>::infinity()) ? v : 0.0f; }

}  // namespace

extern "C" {

// The tap table: 32 x 81 offsets (dx, dy) and distances
int orc_dof_taps(int* dxy, float* d, int mutation) {
    const std::vector<Tap> t = taps_of(mutation);
    for (size_t i = 0; i < t.size(); i++) { dxy[2 * i] = t[i].dx; dxy[2 * i + 1] = t[i].dy; d[i] = t[i].d; }
    return (int)t.size();
}

// The frame's camera ray directions (W x H x 3) of the camera `camera40` (40 floats)
int orc_dof_rays(const float* camera40, int W, int H, float* out) {
    Camera cam; std::memcpy(&cam, camera40, 160);
    for (int y = 0; y < H; y++)
        for (int x = 0; x < W; x++) {
            const V3 d = camera_ray(cam, uv2((u32)x, (u32)y)).dir;
            float* o = out + 3 * ((size_t)y * W + x);
            o[0] = d.x; o[1] = d.y; o[2] = d.z;
        }
    return 0;
}

// Reference mode's lens {h, F, right.xyz, up.xyz, fwd.xyz} of the settings `lens` and the camera; returns whether it is a lens
int orc_dof_lens(const float* lens, const float* transform16, const float* projection16, float* out) {
    return lens_of(lens, transform16, projection16, out);
}

// The thin-lens rays (origins, then directions, W x H x 3 each) of the camera `camera40` with the lens `L` (orc_dof_lens) and seed
int orc_dof_lens_rays(const float* camera40, int W, int H, const float* L, uint32_t seed, float* origins, float* dirs) {
    Camera cam; std::memcpy(&cam, camera40, 160);
    for (int y = 0; y < H; y++)
        for (int x = 0; x < W; x++) {
            const Ray r = lens_ray(cam, L, seed, uv2((u32)x, (u32)y));
            const size_t i = 3 * ((size_t)y * W + x);
            origins[i] = r.origin.x; origins[i + 1] = r.origin.y; origins[i + 2] = r.origin.z;
            dirs[i] = r.dir.x; dirs[i + 1] = r.dir.y; dirs[i + 2] = r.dir.z;
        }
    return 0;
}

// A Reference-mode frame of camera `cam` of the oracle engine `e` (an orc_engine_create handle, procedural sky), as its own schedule
// renders it but with the depth-0 rays of K1 and K2 leaving the thin lens of the settings `lens`; returns 1 when the lens applied
// (F > f), 0 when the camera rendered through the pinhole (the engine's own render)
int orc_dof_render_reference(void* e, int cam, const float* lens, int mutation) {
    Engine* en = (Engine*)e;
    Engine::Cam* c = en->cameras[cam];
    float L[11];
    if (c->cam.mode != MODE_REFERENCE || !lens_of(lens, &c->cam.transform.c[0].x, &c->cam.projection.c[0].x, L)) { en->render_camera(cam); return 0; }
    en->run_atmosphere();
    CamState& cs = c->st;
    const Scene sc = en->scene();
    const u32 f = c->frame;
    const bool alt = (f % 2) == 1;
    auto seed = [&](u32 k) { return dispatch_seed(en->seed_base, f, k); };
    const u32 lseed = mutation == DM_LENS_SHADING_STREAM ? seed(D_REF_SHADING) : seed(kLensDispatch);
    for (u32 d = 0; d <= c->cam.ref_depth; d++) {
        const u32 sd = seed(D_REF_SHADING + d);
        ref_tracing_lens(cs, sc, d, L, lseed);
        ref_shading_lens(cs, sc, sd, d, L, lseed);
    }
    pass_ref_shading(cs, sc, seed(D_REF_SHADING + 31), 255);
    pass_frame_composition(cs, alt, 6, false, false);
    return 1;
}

// lens = {focal_distance, aperture_f_stops, sensor_height, max_radius}; out = {f, A, k, F, R, forward.xyz}
int orc_dof_consts(const float* lens, const float* transform16, const float* projection16, int H, float* out) {
    return consts_of(lens, transform16, projection16, H, out);
}

// The "depth_of_field" words (16 + W H + TX TY) and the defocused frame (W x H x 4) of `output` (W x H x 4) with primary hit distances
// `t` (W x H; 0 on a miss) through the camera `camera40` (the GpuCamera of the frame, 40 floats)
int orc_dof_run(const float* output, const float* t, const float* camera40, int W, int H, const float* lens, const float* transform16,
                const float* projection16, float* words, float* frame, int mutation) {
    static_assert(sizeof(Camera) == 160, "camera layout");
    Camera cam; std::memcpy(&cam, camera40, 160);
    float c[8];
    const int active = consts_of(lens, transform16, projection16, H, c);
    const float k = c[2], F = c[3], R = c[4];
    const V3 fwd = v3(c[5], c[6], c[7]);
    const int TX = (W + kTile - 1) / kTile, TY = (H + kTile - 1) / kTile;
    const size_t n = (size_t)W * H;
    uint32_t head[kHeader] = {(uint32_t)W, (uint32_t)H, (uint32_t)TX, (uint32_t)TY, (uint32_t)active};
    std::memcpy(head + 5, c, sizeof c);
    std::memcpy(words, head, sizeof head);
    float* r = words + kHeader;
    uint32_t* rho_t = (uint32_t*)(r + n);
#pragma omp parallel for schedule(static)
    for (long p = 0; p < (long)n; p++) {
        const int x = (int)(p % W), y = (int)(p / W);
        float v = 0.0f;
        if (active) {
            const float tt = t[p];
            if (tt == 0.0f) v = mutation == DM_SKY_IN_FOCUS ? 0.0f : (k < R ? k : R);
            else {
                const V3 d = camera_ray(cam, uv2((u32)x, (u32)y)).dir;
                const float z = mutation == DM_RAY_DISTANCE ? tt : tt * ((d.x * fwd.x + d.y * fwd.y) + d.z * fwd.z);
                v = mutation == DM_SIGN ? k * (F - z) / z : k * (z - F) / z;
                v = v < -R ? -R : (v > R ? R : v);
            }
        }
        r[p] = v;
    }
    std::vector<float> m((size_t)TX * TY, 0.0f);
    for (size_t p = 0; p < n; p++) {
        const size_t tile = (p / W / kTile) * TX + (p % W) / kTile;
        const float a = std::fabs(r[p]);
        if (a > m[tile]) m[tile] = a;
    }
    const int reach = (int)std::ceil((double)R / kTile);
    for (int ty = 0; ty < TY; ty++)
        for (int tx = 0; tx < TX; tx++) {
            float M = 0.0f;
            const int q = mutation == DM_NO_DILATION ? 0 : reach;
            for (int uy = ty - q; uy <= ty + q; uy++)
                for (int ux = tx - q; ux <= tx + q; ux++)
                    if (ux >= 0 && uy >= 0 && ux < TX && uy < TY && m[(size_t)uy * TX + ux] > M) M = m[(size_t)uy * TX + ux];
            rho_t[(size_t)ty * TX + tx] = M < 0.5f ? 0u : (uint32_t)std::ceil(M);
        }
    const std::vector<Tap> taps = taps_of(mutation);
    auto cl = [](int v, int hi) { return v < 0 ? 0 : (v > hi ? hi : v); };
#pragma omp parallel for schedule(static)
    for (long p = 0; p < (long)n; p++) {
        const int x = (int)(p % W), y = (int)(p / W);
        const int rho = (int)rho_t[(size_t)(y / kTile) * TX + x / kTile];
        float* o = frame + 4 * p;
        if (rho == 0) { std::memcpy(o, output + 4 * p, 16); continue; }
        const float rp = r[p];
        float ax = 0.0f, ay = 0.0f, az = 0.0f, ws = 0.0f;
        for (int i = 0; i < kTaps; i++) {
            const Tap& tp = taps[(size_t)(rho - 1) * kTaps + i];
            const size_t q = (size_t)cl(y + tp.dy, H - 1) * W + cl(x + tp.dx, W - 1);
            const float rq = r[q];
            const float aq = std::fabs(rq), ap = std::fabs(rp);
            const float s = (rq > rp && mutation != DM_NO_BACKGROUND_LIMIT) ? (aq < ap ? aq : ap) : aq;
            float cw = (s - tp.d) + 1.0f;
            cw = cw < 0.0f ? 0.0f : (cw > 1.0f ? 1.0f : cw);
            const float mm = s > 0.5f ? s : 0.5f;
            const float w = mutation == DM_NO_DENSITY ? cw : cw / (mm * mm);
            const float* cq = output + 4 * q;
            ax = ax + finite_or_0(cq[0], mutation) * w; ay = ay + finite_or_0(cq[1], mutation) * w; az = az + finite_or_0(cq[2], mutation) * w;
            ws = ws + w;
        }
        o[0] = ax / ws; o[1] = ay / ws; o[2] = az / ws; o[3] = 1.0f;
    }
    return 0;
}

}  // extern "C"
