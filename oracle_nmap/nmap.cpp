// ORACLE EXTENSION — TEST INFRASTRUCTURE ONLY.  Normal mapping (ST_OPT_NORMAL_MAPS) for the CPU oracle.
//
// The oracle in oracle/ restates the reference, which never reads normal maps, and stays exactly as it is.  This library is that
// oracle (oracle.cpp compiled unchanged into this translation unit) plus one C function, orc_nmap_apply, which restates the
// normal-mapping rule (DESIGN.md §2 "Normal maps"; the formula strolle-gpu/src/material.rs:105-140 keeps commented out) with the
// oracle's own arithmetic and applies it at the three hit-shading sites right after the pass that produced the hit:
//   K0  prim_gbuffer   -> the normal of prim_gbuffer_d0[cur] and prim_surface_map[cur]
//   K12 gi_sampling_a  -> the normal of the packed bounce hit in gi_d1
//   K1  ref_tracing    -> the normal of the packed hit in ref_hits
// Each of those passes stores the hit normal only through normal_encode, and nothing else in the pass depends on it, so re-tracing
// the pass's ray (same ray, same BVH: same triangle) and overwriting the two encoded components gives exactly what the pass would
// have stored with the mapped normal.  oracle_nmap/pyoracle_nmap.py steps a frame pass by pass and calls it after those passes.
#include "../oracle/oracle.cpp"

namespace {
using namespace orc;

// Test-only mistakes (tests/test_normal_maps.py shows that the float64 check catches each): 0 = the rule.
enum { MUT_NONE = 0, MUT_SRGB = 1, MUT_CROSS_ORDER = 2, MUT_NO_BACKFACE_SIGN = 3, MUT_RENORMALISE_T = 4, MUT_NO_FALLBACK = 5 };

// Möller–Trumbore for one triangle and one ray, as triangle_hit (orc_gpu.hpp) computes it: the barycentrics and 1 / det of the hit
// ray_trace accepted on this triangle (same expressions, same operation order, so the same bits).
bool barycentrics(const V4* t, const Ray& ray, float* u_out, float* v_out, float* inv_det_out) {
    V3 p0 = xyz(t[0]), p1 = xyz(t[3]), p2 = xyz(t[6]);
    V3 v0v1 = p1 - p0, v0v2 = p2 - p0;
    V3 pvec = cross(ray.dir, v0v2);
    float det = dot(v0v1, pvec);
    if (abs_(det) < F32_EPSILON) return false;
    float inv_det = 1.0f / det;
    V3 tvec = ray.origin - p0;
    *u_out = dot(tvec, pvec) * inv_det;
    V3 qvec = cross(tvec, v0v1);
    *v_out = dot(ray.dir, qvec) * inv_det;
    *inv_det_out = inv_det;
    return true;
}

// The rule for a closest hit `h` of `ray` (h.normal = triangle_hit's interpolated, sign-flipped normal).
V3 mapped_normal(const Scene& sc, const Ray& ray, const TriangleHit& h, int mutation) {
    const V4 rect = sc.materials[h.material_id].normal_map_texture;
    if (is_zero(rect) || !sc.atlas) return h.normal;
    const V4* t = sc.triangles + 9 * (size_t)h.triangle_id;
    float u, v, inv_det;
    if (!barycentrics(t, ray, &u, &v, &inv_det)) return h.normal;
    const float s = copysign_(1.0f, inv_det);
    const V3 n = h.normal * s;                                  // before the sign flip (exact: the factor is +-1)
    const float w = (1.0f - u) - v;
    const V4 t0 = t[2], t1 = t[5], t2 = t[8];
    V3 tv = (xyz(t1) * u + xyz(t2) * v) + xyz(t0) * w;          // not renormalised (mikktspace)
    const float tw = (t1.w * u + t2.w * v) + t0.w * w;
    if (mutation == MUT_RENORMALISE_T) tv = normalize(tv);
    const V3 b = (mutation == MUT_CROSS_ORDER ? cross(tv, n) : cross(n, tv)) * tw;
    // sample_atlas's wrap, rect mapping and nearest texel (orc_gpu.hpp material_sample_atlas / atlas_fetch), decoded linearly
    const V2 uv = v2(rect.x + wrap_uv(h.uv.x) * rect.z, rect.y + wrap_uv(h.uv.y) * rect.w);
    i32 x = f2i_sat(floor_(uv.x * (float)ATLAS_SIZE)), y = f2i_sat(floor_(uv.y * (float)ATLAS_SIZE));
    if (x < 0) x = 0; if (x > (i32)ATLAS_SIZE - 1) x = (i32)ATLAS_SIZE - 1;
    if (y < 0) y = 0; if (y > (i32)ATLAS_SIZE - 1) y = (i32)ATLAS_SIZE - 1;
    const uint8_t* p = sc.atlas + 4 * ((size_t)y * ATLAS_SIZE + (size_t)x);
    float c[3];
    for (int k = 0; k < 3; k++) c[k] = mutation == MUT_SRGB ? sc.srgb_lut[p[k]] : (float)p[k] / 255.0f;
    const V3 nt = v3(2.0f * c[0] - 1.0f, 2.0f * c[1] - 1.0f, 2.0f * c[2] - 1.0f);
    const V3 m = normalize((tv * nt.x + b * nt.y) + n * nt.z);
    const bool ok = mutation == MUT_NO_FALLBACK || (std::isfinite(m.x) && std::isfinite(m.y) && std::isfinite(m.z) && dot(m, n) > 0.0f);
    const V3 r = ok ? m : n;
    return mutation == MUT_NO_BACKFACE_SIGN ? r : r * s;
}

void patch_normal(V4& texel, int ix, int iy, V3 normal) { V2 e = normal_encode(normal); (&texel.x)[ix] = e.x; (&texel.x)[iy] = e.y; }

}  // namespace

extern "C" {

// Applies the rule to what step `pass` (the device's PassId: 0 = K0, 8 = K12, 21 = K1) of camera `cam`'s current frame just stored;
// `depth` = K1's bounce depth.  Call it right after that step (render_range), before any later step reads its output.
int orc_nmap_apply(void* e, int cam, int pass, int depth, int mutation) {
    Engine* en = (Engine*)e;
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
            V3 n = mapped_normal(sc, ray, th, mutation);
            patch_normal(at(cs.prim_gbuffer_d0[cur], cs.w, p), 1, 2, n);   // gbuffer_pack: d0 = (depth, oct n, bytes)
            patch_normal(at(cs.prim_surface_map[cur], cs.w, p), 0, 1, n);  // (oct n, depth, roughness)
        }
        return 0;
    }
    if (pass == 8) {   // pass_gi_sampling_a's rays (orc_passes.hpp): the direction it stored in gi_d0, the origin it started from
        const bool tracing = frame_is_gi_tracing(f);
        ORC_FOR_HALF_GRID(cs) {
            UV2 gid = uv2(gx_, gy_);
            UV2 sp = tracing ? resolve_checkerboard(gid, f / 2) : resolve_checkerboard(gid, f);
            size_t idx = camera_screen_to_idx(camera, sp);
            if (!camera_contains(camera, sp)) continue;
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
            patch_normal(at(cs.gi_d1, cs.w, gid), 1, 2, mapped_normal(sc, ray, gh, mutation));
        }
        return 0;
    }
    if (pass == 21) {
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
            TriangleHit h = ray_trace(ray, sc);
            if (!trihit_is_some(h)) continue;
            patch_normal(cs.ref_hits[2 * idx + 1], 0, 1, mapped_normal(sc, ray, h, mutation));   // trihit_pack: d1 = (oct n, uv)
        }
        return 0;
    }
    return -1;
}

}  // extern "C"
