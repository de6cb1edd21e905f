// ORACLE — TEST INFRASTRUCTURE ONLY (see orc_math.hpp header).
//
// Restatement of the host slice of the `strolle` crate that the hot path
// depends on: BVH builder + serializer, triangle baking, scene stores
// (materials / lights / instances / triangles), Camera::serialize, atmosphere
// LUT generation, and the per-frame pass schedule of CameraController::render.
#pragma once
#include <algorithm>
#include <functional>
#include <deque>
#include <map>
#include <string>
#include <vector>
#include "orc_passes.hpp"

namespace orc {

// ---------------------------------------------------------------------------
// BoundingBox (strolle/src/utils/bounding_box.rs:5-105)
// ---------------------------------------------------------------------------
struct BBox {
    V3 mn, mx;
    BBox() : mn(v3s(F32_MAX)), mx(v3s(-F32_MAX)) {}
    V3 extent() const { return mx - mn; }
    float half_area() const { V3 e = extent(); return e.x * e.y + e.y * e.z + e.z * e.x; }
    bool is_set() const { return mn.x != F32_MAX; }
    void add(V3 p) { mn = vmin(mn, p); mx = vmax(mx, p); }
    void add(const BBox& b) { add(b.mn); add(b.mx); }
};

// Allocator (strolle/src/utils/allocator.rs:4-58)
struct Allocator {
    std::vector<std::pair<size_t, size_t>> slots;
    bool dirty = false;
    void give(size_t s, size_t e) {
        if (!slots.empty()) dirty |= s <= slots.back().second;
        slots.push_back({s, e});
    }
    bool take(size_t len, size_t* s, size_t* e) {
        compact();
        for (size_t i = 0; i < slots.size(); i++) {
            if (slots[i].second - slots[i].first >= len) {
                size_t remaining = (slots[i].second - slots[i].first) - len;
                if (remaining > 0) { slots[i].first += len; *s = slots[i].first - len; *e = slots[i].first; }
                else { *s = slots[i].first; *e = slots[i].second; slots.erase(slots.begin() + i); }
                return true;
            }
        }
        return false;
    }
    void compact() {
        bool d = dirty; dirty = false;
        if (!d || slots.empty()) return;
        std::stable_sort(slots.begin(), slots.end(), [](const std::pair<size_t, size_t>& a, const std::pair<size_t, size_t>& b) { return a.first < b.first; });
        size_t idx = 0;
        while (idx < slots.size() - 1) {
            if (slots[idx].second == slots[idx + 1].first) { slots[idx].second = slots[idx + 1].second; slots.erase(slots.begin() + idx + 1); }
            else idx++;
        }
    }
};

// ---------------------------------------------------------------------------
// BVH (strolle/src/bvh/*.rs)
// ---------------------------------------------------------------------------
struct BvhPrimitive { u32 triangle_id, material_id; V3 center; BBox bounds; bool alive() const { return center.x != F32_MAX; } };
struct BvhNode { bool internal; BBox bounds; u32 start, end; u32 left_id, right_id; uint64_t left_hash, right_hash; };

// fxhash 0.2.1 (crates.io, Cargo.lock; not vendored) FxHasher on a 64-bit target, restated from its published
// definition: hash = (hash.rotate_left(5) ^ word) * 0x517cc1b727220a95 per written word; write_u32 widens to u64.
struct FxHasher64 {
    uint64_t h = 0;
    void write_u32(u32 w) { h = (((h << 5) | (h >> 59)) ^ (uint64_t)w) * 0x517cc1b727220a95ull; }
    // impl Hash for BvhPrimitive (strolle/src/bvh/primitive.rs:27-37): ONLY the centre's bits are hashed
    void write(const BvhPrimitive& p) { write_u32(f2u(p.center.x)); write_u32(f2u(p.center.y)); write_u32(f2u(p.center.z)); }
};

struct BvhBuilder {
    static const int BINS = 12;  // strolle/src/bvh/builder.rs:15
    static const u32 NONE = 0xffffffffu;
    std::vector<BvhNode> nodes;
    std::vector<BvhPrimitive> prims;  // "current"
    std::vector<BvhNode> prev_nodes;       // last refresh's tree: the "ghost" nodes of builder.rs:245-275
    std::vector<BvhPrimitive> prev_prims;  // BvhPrimitives::previous (primitives.rs:63-65)
    bool reuse = true;                     // false: every refresh builds from scratch (what a first build does)
    u32 reused_subtrees = 0;
    struct Plane { int axis; float at, cost; };
    struct Ref { u32 id, ghost; };         // BvhNodeRef (builder.rs:367-382); ghost = index into prev_nodes

    static float axis_of(V3 v, int a) { return a == 0 ? v.x : (a == 1 ? v.y : v.z); }

    // builder.rs:70-181
    bool find_splitting_plane(u32 node_id, Plane* out) {
        const BvhNode& node = nodes[node_id];
        u32 n = node.end - node.start;
        if (n <= 1) return false;
        const BvhPrimitive* p = prims.data() + node.start;
        BBox cbb;
        for (u32 i = 0; i < n; i++) cbb.add(p[i].center);
        struct Bin { BBox bounds; u32 count; Bin() : count(0) {} };
        Bin bins[3][BINS];
        V3 scale = (float)BINS / cbb.extent();
        for (u32 i = 0; i < n; i++) {
            V3 b = scale * (p[i].center - cbb.mn);
            u32 ix = std::min(f2u_sat(b.x), (u32)BINS - 1), iy = std::min(f2u_sat(b.y), (u32)BINS - 1), iz = std::min(f2u_sat(b.z), (u32)BINS - 1);
            bins[0][ix].count += 1; bins[0][ix].bounds.add(p[i].bounds);
            bins[1][iy].count += 1; bins[1][iy].bounds.add(p[i].bounds);
            bins[2][iz].count += 1; bins[2][iz].bounds.add(p[i].bounds);
        }
        float left_areas[3][BINS - 1], right_areas[3][BINS - 1];
        u32 left_counts[3][BINS - 1], right_counts[3][BINS - 1];
        for (int axis = 0; axis < 3; axis++) {
            BBox lbb, rbb; u32 lc = 0, rc = 0;
            for (int i = 0; i < BINS - 1; i++) {
                const Bin& lb = bins[axis][i];
                lc += lb.count; left_counts[axis][i] = lc;
                if (lb.bounds.is_set()) lbb.add(lb.bounds);
                left_areas[axis][i] = lbb.half_area();
                const Bin& rb = bins[axis][BINS - 1 - i];
                rc += rb.count; right_counts[axis][BINS - 2 - i] = rc;
                if (rb.bounds.is_set()) rbb.add(rb.bounds);
                right_areas[axis][BINS - 2 - i] = rbb.half_area();
            }
        }
        bool have = false; Plane best = {0, 0, 0};
        V3 scale2 = cbb.extent() / (float)BINS;
        for (int axis = 0; axis < 3; axis++) {
            for (int i = 0; i < BINS - 1; i++) {
                float cost = (float)left_counts[axis][i] * left_areas[axis][i] + (float)right_counts[axis][i] * right_areas[axis][i];
                bool better = !have || (cost <= best.cost);
                if (better) {
                    best.axis = axis;
                    best.at = axis_of(cbb.mn, axis) + axis_of(scale2, axis) * (float)(i + 1);
                    best.cost = cost; have = true;
                }
            }
        }
        *out = best;
        return have;
    }
    // builder.rs:321-359 `copy` + `offset_primitives`: the previous subtree rooted at prev_nodes[prev_id] is taken over as it
    // was (node bounds, split structure AND its primitives in their previous order, whatever their other fields are now).
    u32 copy_subtree(u32 prev_id, i32 offset) {
        BvhNode n = prev_nodes[prev_id];
        n.start = (u32)((i32)n.start + offset); n.end = (u32)((i32)n.end + offset);
        u32 id = (u32)nodes.size(); nodes.push_back(n);
        if (n.internal) {
            u32 l = copy_subtree(prev_nodes[prev_id].left_id, offset), r = copy_subtree(prev_nodes[prev_id].right_id, offset);
            nodes[id].left_id = l; nodes[id].right_id = r;
        }
        return id;
    }
    u32 adopt(u32 prev_id, u32 new_start) {
        const BvhNode& pn = prev_nodes[prev_id];
        for (u32 i = pn.start; i < pn.end; i++) prims[new_start + (i - pn.start)] = prev_prims[i];   // primitives.rs:52-59
        reused_subtrees += 1;
        return copy_subtree(prev_id, (i32)new_start - (i32)pn.start);
    }
    // builder.rs:183-319
    void split(const Ref& ref, const Plane& plane, Ref* left, Ref* right) {
        BvhNode node = nodes[ref.id];
        BvhPrimitive* data = prims.data() + node.start;
        i32 l = 0, r = (i32)(node.end - node.start) - 1;
        BBox lb, rb;
        FxHasher64 lh, rh;
        while (l <= r) {
            BvhPrimitive pr = data[l];
            if (axis_of(pr.center, plane.axis) < plane.at) { l += 1; lb.add(pr.bounds); lh.write(pr); }
            else { std::swap(data[l], data[r]); r -= 1; rb.add(pr.bounds); rh.write(pr); }
        }
        u32 pivot = node.start + (u32)l;
        u32 left_id = NONE, right_id = NONE;
        left->ghost = right->ghost = NONE;
        bool left_continue = true, right_continue = true;
        if (reuse && ref.ghost != NONE && prev_nodes[ref.ghost].internal) {
            const BvhNode g = prev_nodes[ref.ghost];
            if (g.left_hash == lh.h) { left_id = adopt(g.left_id, node.start); left_continue = false; } else left->ghost = g.left_id;
            if (g.right_hash == rh.h) { right_id = adopt(g.right_id, pivot); right_continue = false; } else right->ghost = g.right_id;
        }
        if (left_id == NONE) {
            BvhNode ln; ln.internal = false; ln.bounds = lb; ln.start = node.start; ln.end = pivot; ln.left_id = ln.right_id = 0; ln.left_hash = ln.right_hash = 0;
            nodes.push_back(ln); left_id = (u32)nodes.size() - 1;
        }
        if (right_id == NONE) {
            BvhNode rn; rn.internal = false; rn.bounds = rb; rn.start = pivot; rn.end = node.end; rn.left_id = rn.right_id = 0; rn.left_hash = rn.right_hash = 0;
            nodes.push_back(rn); right_id = (u32)nodes.size() - 1;
        }
        nodes[ref.id].internal = true; nodes[ref.id].left_id = left_id; nodes[ref.id].right_id = right_id;
        nodes[ref.id].left_hash = lh.h; nodes[ref.id].right_hash = rh.h;
        left->id = left_continue ? left_id : NONE;
        right->id = right_continue ? right_id : NONE;
    }
    // builder.rs:17-67 + Bvh::refresh (bvh.rs:48-70): begin_refresh, build, (serialize), end_refresh
    void run(const std::vector<BvhPrimitive>& all) {
        prev_nodes.swap(nodes); prev_prims.swap(prims);   // what end_refresh left behind
        prims.clear();
        for (const BvhPrimitive& p : all) if (p.alive()) prims.push_back(p);   // primitives.rs:58-61
        nodes.clear();
        reused_subtrees = 0;
        BvhNode root; root.internal = false; root.bounds = BBox(); root.start = 0; root.end = (u32)prims.size(); root.left_id = root.right_id = 0; root.left_hash = root.right_hash = 0;
        nodes.push_back(root);
        std::deque<Ref> queue; queue.push_back(Ref{0, prev_nodes.empty() ? NONE : 0u});
        while (!queue.empty()) {
            Ref ref = queue.front(); queue.pop_front();
            Plane plane;
            if (find_splitting_plane(ref.id, &plane)) {
                float sah = (float)(nodes[ref.id].end - nodes[ref.id].start) * nodes[ref.id].bounds.half_area();  // node.rs:36-46
                if (plane.cost < sah) {
                    Ref l, r; split(ref, plane, &l, &r);
                    if (l.id != NONE) queue.push_back(l);
                    if (r.id != NONE) queue.push_back(r);
                }
            }
        }
    }
    // serializer.rs:20-110
    u32 serialize(std::vector<V4>& buf, const std::vector<uint8_t>& material_alpha_blend, u32 id, int depth, int* max_depth) const {
        u32 ptr = (u32)buf.size();
        if (depth > *max_depth) *max_depth = depth;
        const BvhNode& n = nodes[id];
        if (n.internal) {
            for (int i = 0; i < 4; i++) buf.push_back(v4z());
            BBox lb = nodes[n.left_id].bounds, rb = nodes[n.right_id].bounds;
            serialize(buf, material_alpha_blend, n.left_id, depth + 1, max_depth);
            u32 right_ptr = serialize(buf, material_alpha_blend, n.right_id, depth + 1, max_depth);
            buf[ptr] = v4(lb.mn, u2f(0));
            buf[ptr + 1] = v4(lb.mx, u2f(right_ptr));
            buf[ptr + 2] = v4(rb.mn, 0.0f);
            buf[ptr + 3] = v4(rb.mx, 0.0f);
        } else {
            u32 cnt = n.end - n.start;
            for (u32 i = 0; i < cnt; i++) {
                const BvhPrimitive& p = prims[n.start + i];
                u32 flags = ((i + 1 < cnt) ? 1u : 0u) | ((material_alpha_blend[p.material_id] ? 1u : 0u) << 1);
                buf.push_back(v4(u2f(flags), u2f(p.triangle_id), u2f(p.material_id), u2f(1)));
            }
        }
        return ptr;
    }
};

// ---------------------------------------------------------------------------
// Mesh triangles (strolle/src/mesh_triangle.rs:47-86, triangle.rs:16-38)
// ---------------------------------------------------------------------------
struct Affine { V3 x, y, z, t; };  // glam Affine3A: matrix3 columns + translation
static inline V3 affine_point(const Affine& a, V3 p) { return ((a.x * p.x + a.y * p.y) + a.z * p.z) + a.t; }   // Affine3A::transform_point3
static inline V3 mat3_mul(const Affine& a, V3 v) { return (a.x * v.x + a.y * v.y) + a.z * v.z; }
static inline float mat3_det(const Affine& a) { return dot(a.z, cross(a.x, a.y)); }
static inline Affine affine_inverse(const Affine& a) {  // glam Affine3A::inverse (Mat3A::inverse + -(m^-1 * t))
    V3 tmp0 = cross(a.y, a.z), tmp1 = cross(a.z, a.x), tmp2 = cross(a.x, a.y);
    float det = dot(a.z, tmp2);
    V3 inv_det = v3s(1.0f / det);
    // transpose of (tmp0*inv_det, tmp1*inv_det, tmp2*inv_det)
    V3 c0 = tmp0 * inv_det, c1 = tmp1 * inv_det, c2 = tmp2 * inv_det;
    Affine r;
    r.x = v3(c0.x, c1.x, c2.x); r.y = v3(c0.y, c1.y, c2.y); r.z = v3(c0.z, c1.z, c2.z);
    r.t = -mat3_mul(r, a.t);
    return r;
}
struct MeshTriangle { V3 positions[3], normals[3]; V2 uvs[3]; V4 tangents[3]; };
static inline MeshTriangle mesh_triangle_build(const MeshTriangle& in, const Affine& xf, const Affine& xf_inv) {
    MeshTriangle out;
    // Mat4::from(xform_inv).transpose().transform_vector3(n): rows of xf_inv's 3x3 become columns
    Affine tr; tr.x = v3(xf_inv.x.x, xf_inv.y.x, xf_inv.z.x); tr.y = v3(xf_inv.x.y, xf_inv.y.y, xf_inv.z.y); tr.z = v3(xf_inv.x.z, xf_inv.y.z, xf_inv.z.z); tr.t = v3s(0);
    float sign = (f2u(mat3_det(xf)) >> 31) ? -1.0f : 1.0f;
    for (int i = 0; i < 3; i++) {
        out.positions[i] = affine_point(xf, in.positions[i]);
        out.normals[i] = normalize(mat3_mul(tr, in.normals[i]));
        V3 tg = normalize(mat3_mul(xf, xyz(in.tangents[i])));
        out.tangents[i] = v4(tg, in.tangents[i].w * sign);
        out.uvs[i] = in.uvs[i];
    }
    return out;
}
static inline V3 triangle_center(const MeshTriangle& t) { return ((v3s(0) + t.positions[0]) + t.positions[1] + t.positions[2]) / 3.0f; }  // iter().sum() starts from zero
static inline void triangle_serialize(const MeshTriangle& t, V4* out9) {
    for (int i = 0; i < 3; i++) { out9[3 * i] = v4(t.positions[i], t.uvs[i].x); out9[3 * i + 1] = v4(t.normals[i], t.uvs[i].y); out9[3 * i + 2] = t.tangents[i]; }
}

// Camera::serialize (strolle/src/camera.rs:50-66)
static inline Camera camera_serialize(const M4& transform, const M4& projection, u32 w, u32 h) {
    Camera c;
    c.projection_view = mul(projection, inverse(transform));
    c.ndc_to_world = mul(transform, inverse(projection));
    c.origin = v4(transform.c[3].x, transform.c[3].y, transform.c[3].z, 0.0f);   // to_scale_rotation_translation().2
    c.screen = v4((float)w, (float)h, 0.0f, 0.0f);
    return c;
}

// ---------------------------------------------------------------------------
// Atmosphere LUT generation (strolle-shaders/src/atmosphere/*.rs)
// Rgba16Float storage restated as f32 values rounded to binary16 (RNE).
// ---------------------------------------------------------------------------
static inline float round_f16(float f) {
    u32 x = f2u(f);
    u32 sign = x & 0x80000000u; x &= 0x7fffffffu;
    if (x >= 0x7f800000u) return f;                       // inf / nan
    if (x >= 0x477ff000u) return u2f(sign | 0x7f800000u);   // >= 65520 -> inf
    if (x < 0x38800000u) {                                // subnormal half (< 2^-14): quantum 2^-24
        float a = u2f(x);
        float q = a * 16777216.0f;                        // exact
        float r = q - floor_(q);
        float fl = floor_(q);
        if (r > 0.5f || (r == 0.5f && fmod_(fl, 2.0f) != 0.0f)) fl += 1.0f;
        return u2f(sign | f2u(fl * (1.0f / 16777216.0f)));
    }
    u32 lsb = (x >> 13) & 1u;
    x += 0xfffu + lsb;
    x &= 0xffffe000u;
    return u2f(sign | x);
}
static inline void atm_eval_scattering(V3 pos, V3* rayleigh, float* mie, V3* extinction) {  // atmosphere/utils.rs:3-27
    float altitude_km = (length(pos) - ATM_GROUND_RADIUS_MM) * 1000.0f;
    float rayleigh_density = exp_(-altitude_km / 8.0f);
    float mie_density = exp_(-altitude_km / 1.2f);
    V3 rs = v3(5.802f, 13.558f, 33.1f) * rayleigh_density;
    // RAYLEIGH_ABSORPTION_BASE is the constant 0.0: `0.0 * density` is folded to 0 (as GPU shader
    // compilers do).  Evaluated literally it is 0*inf = NaN below ground (density overflows), which
    // poisons the whole sky LUT for a sun below the horizon (DESIGN.md "quirk C-18").
    float ms = 3.996f * mie_density;
    float ma = 4.4f * mie_density;
    V3 oz = v3(0.650f, 1.881f, 0.085f) * fmax_(1.0f - abs_(altitude_km - 25.0f) / 15.0f, 0.0f);
    *rayleigh = rs; *mie = ms;
    *extinction = ((rs + v3s(ms)) + v3s(ma)) + oz;
}
static inline float atm_mie_phase(float cos_theta) {
    const float G = 0.8f; const float SCALE = 3.0f / (8.0f * PI);
    float num = (1.0f - G * G) * (1.0f + cos_theta * cos_theta);
    float denom = (2.0f + G * G) * pow_(1.0f + G * G - 2.0f * G * cos_theta, 1.5f);
    return SCALE * num / denom;
}
static inline float atm_rayleigh_phase(float cos_theta) { const float K = 3.0f / (16.0f * PI); return K * (1.0f + cos_theta * cos_theta); }
static inline V3 vexp(V3 v) { return v3(exp_(v.x), exp_(v.y), exp_(v.z)); }
static inline V3 atm_transmittance_eval(V3 pos, V3 sun_dir) {  // generate_transmittance_lut.rs:29-59
    if (ray_intersect_sphere(ray_new(pos, sun_dir), ATM_GROUND_RADIUS_MM) > 0.0f) return v3s(0);
    float atmosphere_distance = ray_intersect_sphere(ray_new(pos, sun_dir), ATM_ATMOSPHERE_RADIUS_MM);
    float t = 0.0f; V3 transmittance = v3s(1.0f);
    for (float i = 0.0f; i < 40.0f; i += 1.0f) {
        float new_t = ((i + 0.3f) / 40.0f) * atmosphere_distance;
        float dt = new_t - t; t = new_t;
        V3 new_pos = pos + t * sun_dir;
        V3 rs, ext; float ms; atm_eval_scattering(new_pos, &rs, &ms, &ext);
        transmittance *= vexp(-dt * ext);
    }
    return transmittance;
}
struct AtmosphereLuts { std::vector<V4> transmittance, scattering, sky; float sky_altitude; bool have_static, have_sky; AtmosphereLuts() : sky_altitude(0), have_static(false), have_sky(false) {} };
static void atm_generate_transmittance(std::vector<V4>& out) {  // 256x64
    out.assign(256 * 64, v4z());
    _Pragma("omp parallel for") for (int y = 0; y < 64; y++) for (int x = 0; x < 256; x++) {
        V2 uv = v2((float)x, (float)y) / v2(256.0f, 64.0f);
        float sun_cos_theta = 2.0f * uv.x - 1.0f;
        float sun_theta = acos_(clampf(sun_cos_theta, -1.0f, 1.0f));
        float height = lerp_c(ATM_GROUND_RADIUS_MM, ATM_ATMOSPHERE_RADIUS_MM, uv.y);
        V3 pos = v3(0.0f, height, 0.0f);
        V3 sun_dir = normalize(v3(0.0f, sun_cos_theta, -sin_(sun_theta)));
        V3 v = atm_transmittance_eval(pos, sun_dir);
        out[(size_t)y * 256 + x] = v4(round_f16(v.x), round_f16(v.y), round_f16(v.z), 1.0f);
    }
}
static void atm_generate_scattering(const std::vector<V4>& trans, std::vector<V4>& out) {  // 32x32, generate_scattering_lut.rs
    out.assign(32 * 32, v4z());
    Lut tl = {256, 64, trans.data()};
    _Pragma("omp parallel for") for (int y = 0; y < 32; y++) for (int x = 0; x < 32; x++) {
        V2 uv = v2((float)x, (float)y) / v2(32.0f, 32.0f);
        float sun_cos_theta = 2.0f * uv.x - 1.0f;
        float sun_theta = acos_(clampf(sun_cos_theta, -1.0f, 1.0f));
        float height = lerp_c(ATM_GROUND_RADIUS_MM, ATM_ATMOSPHERE_RADIUS_MM, fmax_(uv.y, 0.01f));
        V3 pos = v3(0.0f, height, 0.0f);
        V3 sun_dir = normalize(v3(0.0f, sun_cos_theta, -sin_(sun_theta)));
        V3 lum_total = v3s(0), fms = v3s(0);
        const int S = 8;
        float inv_samples = 1.0f / (float)(S * S);
        for (int i = 0; i < S; i++) for (int j = 0; j < S; j++) {
            float theta = PI * ((float)i + 0.5f) / (float)S;
            float phi = acos_(clampf(1.0f - 2.0f * ((float)j + 0.5f) / (float)S, -1.0f, 1.0f));
            float cos_phi = cos_(phi), sin_phi = sin_(phi), cos_th = cos_(theta), sin_th = sin_(theta);
            V3 ray_dir = v3(sin_phi * sin_th, cos_phi, sin_phi * cos_th);
            float atmosphere_distance = ray_intersect_sphere(ray_new(pos, ray_dir), ATM_ATMOSPHERE_RADIUS_MM);
            float ground_distance = ray_intersect_sphere(ray_new(pos, ray_dir), ATM_GROUND_RADIUS_MM);
            float t_max = (ground_distance > 0.0f) ? ground_distance : atmosphere_distance;
            float cos_theta = dot(ray_dir, sun_dir);
            float mie_phase = atm_mie_phase(cos_theta), rayleigh_phase = atm_rayleigh_phase(-cos_theta);
            V3 lum = v3s(0), lum_factor = v3s(0), transmittance = v3s(1.0f);
            float t = 0.0f;
            for (float step_i = 0.0f; step_i < 20.0f; step_i += 1.0f) {
                float new_t = ((step_i + 0.3f) / 20.0f) * t_max;
                float dt = new_t - t; t = new_t;
                V3 new_pos = pos + t * ray_dir;
                V3 rs, ext; float ms; atm_eval_scattering(new_pos, &rs, &ms, &ext);
                V3 sample_transmittance = vexp(-dt * ext);
                V3 scattering_no_phase = rs + v3s(ms);
                V3 scattering_f = (scattering_no_phase - scattering_no_phase * sample_transmittance) / ext;
                lum_factor += transmittance * scattering_f;
                V3 sun_transmittance = atm_sample_lut(tl, new_pos, sun_dir);
                V3 rayleigh_in = rs * rayleigh_phase;
                float mie_in = ms * mie_phase;
                V3 in_scattering = (rayleigh_in + v3s(mie_in)) * sun_transmittance;
                V3 scattering_integral = (in_scattering - in_scattering * sample_transmittance) / ext;
                lum += scattering_integral * transmittance;
                transmittance *= sample_transmittance;
            }
            if (ground_distance > 0.0f) {
                V3 hit_pos = pos + ground_distance * ray_dir;
                if (dot(pos, sun_dir) > 0.0f) {
                    hit_pos = normalize(hit_pos) * ATM_GROUND_RADIUS_MM;
                    lum += transmittance * v3s(0.25f) * atm_sample_lut(tl, hit_pos, sun_dir);
                }
            }
            fms += lum_factor * inv_samples;
            lum_total += lum * inv_samples;
        }
        V3 o = lum_total / (v3s(1.0f) - fms);
        out[(size_t)y * 32 + x] = v4(round_f16(o.x), round_f16(o.y), round_f16(o.z), 1.0f);
    }
}
static void atm_generate_sky(const std::vector<V4>& trans, const std::vector<V4>& scat, float sun_altitude, std::vector<V4>& out) {  // 256x256, generate_sky_lut.rs
    out.assign(256 * 256, v4z());
    Lut tl = {256, 64, trans.data()}, sl = {32, 32, scat.data()};
    _Pragma("omp parallel for") for (int y = 0; y < 256; y++) for (int x = 0; x < 256; x++) {
        V2 uv = v2((float)x, (float)y) / v2(256.0f, 256.0f);
        float azimuth = (uv.x - 0.5f) * 2.0f * PI;
        float v;
        if (uv.y < 0.5f) { float coord = 1.0f - 2.0f * uv.y; v = -coord * coord; }
        else { float coord = uv.y * 2.0f - 1.0f; v = coord * coord; }
        V3 vp = atm_view_pos();
        float height = length(vp);
        float horizon;
        { float t = sqr(height) - sqr(ATM_GROUND_RADIUS_MM); t = sqrt_(t) / height; horizon = acos_(clampf(t, -1.0f, 1.0f)) - 0.5f * PI; }
        float altitude = v * 0.5f * PI - horizon;
        V3 ray_dir = v3(cos_(altitude) * sin_(azimuth), sin_(altitude), -cos_(altitude) * cos_(azimuth));
        float sa = fmod_(sun_altitude, 2.0f * PI);
        V3 sun_dir = (sa < 0.5f * PI) ? v3(0.0f, sin_(sa), -cos_(sa)) : v3(0.0f, sin_(sa), cos_(sa));
        float atmosphere_distance = ray_intersect_sphere(ray_new(vp, ray_dir), ATM_ATMOSPHERE_RADIUS_MM);
        float ground_distance = ray_intersect_sphere(ray_new(vp, ray_dir), ATM_GROUND_RADIUS_MM);
        float t_max = (ground_distance < 0.0f) ? atmosphere_distance : ground_distance;
        float cos_theta = dot(ray_dir, sun_dir);
        float mie_phase = atm_mie_phase(cos_theta), rayleigh_phase = atm_rayleigh_phase(-cos_theta);
        V3 lum = v3s(0), transmittance = v3s(1.0f);
        float t = 0.0f;
        for (float i = 0.0f; i < 32.0f; i += 1.0f) {
            float new_t = ((i + 0.3f) / 32.0f) * t_max;
            float dt = new_t - t; t = new_t;
            V3 new_pos = vp + t * ray_dir;
            V3 rs, ext; float ms; atm_eval_scattering(new_pos, &rs, &ms, &ext);
            V3 sample_transmittance = vexp(-dt * ext);
            V3 sun_transmittance = atm_sample_lut(tl, new_pos, sun_dir);
            V3 psi_ms = atm_sample_lut(sl, new_pos, sun_dir);
            V3 rayleigh_in = rs * (rayleigh_phase * sun_transmittance + psi_ms);
            V3 mie_in = ms * (mie_phase * sun_transmittance + psi_ms);
            V3 in_scattering = rayleigh_in + mie_in;
            V3 scattering_integral = (in_scattering - in_scattering * sample_transmittance) / ext;
            lum += scattering_integral * transmittance;
            transmittance *= sample_transmittance;
        }
        out[(size_t)y * 256 + x] = v4(round_f16(lum.x), round_f16(lum.y), round_f16(lum.z), 1.0f);
    }
}

// ---------------------------------------------------------------------------
// Explicit per-dispatch seeds.  The reference draws rand::thread_rng() per
// dispatch (strolle/src/camera_controller.rs:189-194) and is therefore not
// reproducible; both oracle and product derive seeds from (base, frame,
// dispatch id) instead (SURVEY §8d).
// ---------------------------------------------------------------------------
enum DispatchId { D_DI_SAMPLING = 1, D_DI_TEMPORAL = 2, D_DI_SPATIAL_PICK = 3, D_DI_SPATIAL_SAMPLE = 5, D_GI_SAMPLING_A = 8, D_GI_SAMPLING_B = 9,
                  D_GI_TEMPORAL = 10, D_GI_SPATIAL_PICK = 11, D_GI_SPATIAL_SAMPLE = 13, D_GI_PREVIEW = 14, D_REF_SHADING = 32 };
static inline u32 dispatch_seed(u32 base, u32 frame, u32 k) {
    u32 s = base ^ (frame * 64u + k);
    s = s * 747796405u + 2891336453u;
    u32 w = ((s >> ((s >> 28) + 4u)) ^ s) * 277803737u;
    return (w >> 22) ^ w;
}

// ---------------------------------------------------------------------------
// Engine mirror (strolle/src/lib.rs:104-395).  Handles are u64; hash maps are
// replaced by insertion-ordered containers (the reference iterates a std
// HashMap, SURVEY §0 — order there is unspecified).
// ---------------------------------------------------------------------------
struct HostMaterial { V4 base_color, emissive; float perceptual_roughness, metallic, reflectance, ior; bool alpha_blend;
                      uint64_t tex[4]; bool has_tex[4];   // base_color, emissive, metallic_roughness, normal_map (strolle/src/material.rs:13-22)
                      HostMaterial() { for (int i = 0; i < 4; i++) { tex[i] = 0; has_tex[i] = false; } } };
struct HostLight { int type; V3 position; float radius; V3 color; float range; V3 direction; float angle; };
enum CamMode { MODE_IMAGE = 0, MODE_DI_DIFFUSE, MODE_DI_SPECULAR, MODE_GI_DIFFUSE, MODE_GI_SPECULAR, MODE_BVH_HEATMAP, MODE_REFERENCE };
struct HostCamera { int mode; bool denoise; u32 ref_depth; u32 w, h; M4 transform, projection; };

struct Engine {
    // meshes
    std::map<uint64_t, std::vector<MeshTriangle>> meshes;
    // materials (strolle/src/materials.rs)
    std::vector<HostMaterial> materials; std::vector<std::pair<uint64_t, u32>> material_index; std::vector<Material> gpu_materials; bool dirty_materials = false;
    // instances + triangles (strolle/src/instances.rs, triangles.rs)
    struct Inst { uint64_t handle, mesh, material; Affine xf, xf_inv, prev_xf; bool dirty; };
    std::vector<Inst> instances; bool dirty_instances = false;
    struct IdxInst { uint64_t handle; size_t s, e; };
    std::vector<IdxInst> tri_index; Allocator tri_alloc; std::vector<V4> gpu_triangles; std::vector<BvhPrimitive> bvh_all;
    BvhBuilder bvh; std::vector<V4> gpu_bvh; int bvh_depth = 0;
    std::vector<u32> tri_instance; std::vector<V4> instance_xforms;
    // lights (strolle/src/lights.rs); handle UINT64_MAX is the sun
    std::vector<Light> lights; std::vector<std::pair<uint64_t, u32>> light_index;
    std::vector<uint64_t> l_created, l_updated; std::vector<std::pair<uint64_t, u32>> l_remapped; std::vector<u32> l_killed; u32 next_light_id = 1;
    std::vector<Light> gpu_lights;   // what the GPU sees this frame (snapshot at flush)
    World world; float sun_azimuth = 0.0f, sun_altitude = 0.35f; bool dirty_sun = true;
    u32 frame = 1;
    std::vector<uint8_t> blue_noise;
    AtmosphereLuts luts;
    u32 seed_base = 0xC0FFEEu;
    // images (strolle/src/images.rs): a shelf allocator stands in for the guillotiere crate (pinned 0.6 in
    // Cargo.lock, not vendored) — rect placement is an implementation detail, only the rect handed to the
    // material (Images::lookup, images.rs:114-123) matters to the shaders
    struct ImageRect { uint64_t handle; u32 x, y, w, h; };
    std::vector<ImageRect> images; u32 shelf_x = 0, shelf_y = 0, shelf_h = 0; bool dirty_images = false;
    std::vector<uint8_t> atlas; std::vector<float> srgb_lut;
    // cameras
    struct Cam { HostCamera cam; CamState st; u32 frame; bool alive; };
    std::vector<Cam*> cameras;

    Engine() { world.light_count = 0; world.sun_azimuth = 0; world.sun_altitude = 0; world._pad = 0; lights.push_back(make_sun(v3s(0), v3s(0))); light_index.push_back({UINT64_MAX, 0}); }
    ~Engine() { for (Cam* c : cameras) delete c; }

    static Light make_sun(V3 pos, V3 color) {  // strolle-gpu/src/light.rs:49-65
        Light l; l.d0 = v4(pos, 25.0f); l.d1 = v4(color, F32_INF); l.d2 = v4(u2f(1), 0, 0, 0); l.d3 = v4z(); l.prev_d0 = l.prev_d1 = l.prev_d2 = v4z(); return l;
    }
    static Light serialize_light(const HostLight& h) {  // strolle/src/light.rs:25-79
        Light l; l.d0 = v4(h.position, h.radius); l.d1 = v4(h.color, h.range);
        if (h.type == 1) l.d2 = v4(u2f(1), 0, 0, 0);
        else { V2 d = normal_encode(h.direction); l.d2 = v4(u2f(2), d.x, d.y, h.angle); }
        l.d3 = v4z(); l.prev_d0 = l.prev_d1 = l.prev_d2 = v4z(); return l;
    }
    u32* find_light(uint64_t h) { for (auto& p : light_index) if (p.first == h) return &p.second; return nullptr; }
    static void uniq_push(std::vector<uint64_t>& v, uint64_t h) { if (std::find(v.begin(), v.end(), h) == v.end()) v.push_back(h); }
    static void uniq_erase(std::vector<uint64_t>& v, uint64_t h) { v.erase(std::remove(v.begin(), v.end(), h), v.end()); }
    void light_update(u32 idx, uint64_t handle, Light nw) {  // lights.rs:168-182
        Light old = lights[idx]; nw.prev_d0 = old.d0; nw.prev_d1 = old.d1; nw.prev_d2 = old.d2;
        uniq_push(l_updated, handle); lights[idx] = nw;
    }
    void insert_light(uint64_t handle, const HostLight& h) {  // lights.rs:54-82
        Light item = serialize_light(h);
        if (u32* id = find_light(handle)) { light_update(*id, handle, item); return; }
        u32 id;
        if (next_light_id < lights.size()) { lights[next_light_id] = item; id = next_light_id; }
        else { id = (u32)lights.size(); lights.push_back(item); }
        light_index.push_back({handle, id});
        uniq_push(l_created, handle);
        next_light_id += 1;
    }
    void remove_light(uint64_t handle) {  // lights.rs:101-127
        u32* idp = find_light(handle); if (!idp) return;
        u32 id = *idp;
        light_index.erase(std::remove_if(light_index.begin(), light_index.end(), [&](const std::pair<uint64_t, u32>& p) { return p.first == handle; }), light_index.end());
        lights.erase(lights.begin() + id);
        Light zero; zero.d0 = zero.d1 = zero.d2 = zero.d3 = zero.prev_d0 = zero.prev_d1 = zero.prev_d2 = v4z(); lights.push_back(zero);
        uniq_erase(l_created, handle); uniq_erase(l_updated, handle);
        l_remapped.erase(std::remove_if(l_remapped.begin(), l_remapped.end(), [&](const std::pair<uint64_t, u32>& p) { return p.first == handle; }), l_remapped.end());
        if (std::find(l_killed.begin(), l_killed.end(), id) == l_killed.end()) l_killed.push_back(id);
        next_light_id -= 1;
        for (auto& p : light_index) if (p.second > id) {
            bool have = false; for (auto& r : l_remapped) if (r.first == p.first) have = true;
            if (!have) l_remapped.push_back({p.first, p.second});
            p.second -= 1;
        }
    }
    void lights_flush() {  // lights.rs:133-162
        for (u32 id : l_killed) lights[id].d3.x = u2f(0xcafebabeu);
        for (auto& r : l_remapped) lights[r.second].d3.x = u2f(*find_light(r.first) + 1u);
        gpu_lights = lights;
        for (uint64_t h : l_created) { Light& l = lights[*find_light(h)]; l.prev_d0 = l.d0; l.prev_d1 = l.d1; l.prev_d2 = l.d2; }
        for (uint64_t h : l_updated) { Light& l = lights[*find_light(h)]; l.prev_d0 = l.d0; l.prev_d1 = l.d1; l.prev_d2 = l.d2; }
        for (u32 id : l_killed) lights[id].d3.x = u2f(0);
        for (auto& r : l_remapped) lights[r.second].d3.x = u2f(0);
        l_created.clear(); l_updated.clear(); l_remapped.clear(); l_killed.clear();
    }
    void update_sun(float az, float alt) { sun_azimuth = az; sun_altitude = alt; dirty_sun = true; }

    bool insert_image(uint64_t h, const uint8_t* rgba, u32 w, u32 hgt) {   // images.rs:54-104 (ImageData::Raw)
        if (atlas.empty()) {
            atlas.assign((size_t)ATLAS_SIZE * ATLAS_SIZE * 4, 0);
            srgb_lut.resize(256);
            for (int i = 0; i < 256; i++) { float c = (float)i / 255.0f; srgb_lut[i] = (c <= 0.04045f) ? c / 12.92f : pow_((c + 0.055f) / 1.055f, 2.4f); }
        }
        ImageRect* r = nullptr;
        for (ImageRect& k : images) if (k.handle == h) r = &k;
        if (!r || r->w != w || r->h != hgt) {
            if (shelf_x + w > ATLAS_SIZE) { shelf_x = 0; shelf_y += shelf_h; shelf_h = 0; }
            if (w > ATLAS_SIZE || shelf_y + hgt > ATLAS_SIZE) return false;   // "no more space in the atlas"
            ImageRect nr = {h, shelf_x, shelf_y, w, hgt};
            shelf_x += w; if (hgt > shelf_h) shelf_h = hgt;
            if (r) *r = nr; else { images.push_back(nr); r = &images.back(); }
        }
        for (u32 y = 0; y < hgt; y++) std::memcpy(&atlas[4 * ((size_t)(r->y + y) * ATLAS_SIZE + r->x)], rgba + 4 * (size_t)y * w, 4 * (size_t)w);
        dirty_images = true;
        return true;
    }
    V4 image_lookup(bool has, uint64_t h) const {   // images.rs:114-127
        if (!has) return v4z();
        for (const ImageRect& k : images) if (k.handle == h)
            return v4((float)k.x / (float)ATLAS_SIZE, (float)k.y / (float)ATLAS_SIZE, (float)k.w / (float)ATLAS_SIZE, (float)k.h / (float)ATLAS_SIZE);
        return v4z();
    }
    void insert_mesh(uint64_t h, const std::vector<MeshTriangle>& tris) { meshes[h] = tris; }
    void insert_material(uint64_t h, const HostMaterial& m) {  // materials.rs:36-55
        for (auto& p : material_index) if (p.first == h) { materials[p.second] = m; dirty_materials = true; return; }
        materials.push_back(m); material_index.push_back({h, (u32)materials.size() - 1}); dirty_materials = true;
    }
    bool lookup_material(uint64_t h, u32* id) { for (auto& p : material_index) if (p.first == h) { *id = p.second; return true; } return false; }
    void insert_instance(uint64_t h, uint64_t mesh, uint64_t material, const Affine& xf) {  // instances.rs:29-50, instance.rs:15-31
        for (Inst& i : instances) if (i.handle == h) { i.prev_xf = i.xf; i.mesh = mesh; i.material = material; i.xf = xf; i.xf_inv = affine_inverse(xf); i.dirty = true; dirty_instances = true; return; }
        Inst i; i.handle = h; i.mesh = mesh; i.material = material; i.xf = xf; i.xf_inv = affine_inverse(xf); i.prev_xf = xf; i.dirty = true;
        instances.push_back(i); dirty_instances = true;
    }
    void triangles_remove(uint64_t h) {  // triangles.rs:157-171
        for (size_t k = 0; k < tri_index.size(); k++) if (tri_index[k].handle == h) {
            tri_alloc.give(tri_index[k].s, tri_index[k].e);
            for (size_t t = tri_index[k].s; t < tri_index[k].e; t++) bvh_all[t].center = v3s(F32_MAX);
            tri_index.erase(tri_index.begin() + k); return;
        }
    }
    void remove_instance(uint64_t h) {  // lib.rs:226-229
        size_t before = instances.size();
        instances.erase(std::remove_if(instances.begin(), instances.end(), [&](const Inst& i) { return i.handle == h; }), instances.end());
        dirty_instances |= instances.size() != before;
        triangles_remove(h);
    }
    void triangles_create(uint64_t h, const std::vector<MeshTriangle>& tris, u32 material_id) {  // triangles.rs:37-126
        size_t s, e;
        if (tri_alloc.take(tris.size(), &s, &e)) {
            for (size_t i = 0; i < tris.size(); i++) {
                triangle_serialize(tris[i], &gpu_triangles[9 * (s + i)]);
                BvhPrimitive p; p.triangle_id = (u32)(s + i); p.material_id = material_id; p.center = triangle_center(tris[i]);
                p.bounds = BBox(); for (int k = 0; k < 3; k++) p.bounds.add(tris[i].positions[k]);
                bvh_all[s + i] = p;
            }
        } else {
            s = gpu_triangles.size() / 9;
            for (size_t i = 0; i < tris.size(); i++) {
                gpu_triangles.resize(gpu_triangles.size() + 9);
                triangle_serialize(tris[i], &gpu_triangles[9 * (s + i)]);
                BvhPrimitive p; p.triangle_id = (u32)(s + i); p.material_id = material_id; p.center = triangle_center(tris[i]);
                p.bounds = BBox(); for (int k = 0; k < 3; k++) p.bounds.add(tris[i].positions[k]);
                bvh_all.push_back(p);
            }
            e = s + tris.size();
        }
        tri_index.push_back({h, s, e});
    }
    bool instances_refresh() {  // instances.rs:69-139
        bool d = dirty_instances; dirty_instances = false;
        if (!d) return false;
        for (Inst& in : instances) {
            bool id = in.dirty; in.dirty = false;
            if (!id) continue;
            auto mit = meshes.find(in.mesh);
            u32 material_id;
            if (mit == meshes.end() || !lookup_material(in.material, &material_id)) { in.dirty = true; dirty_instances = true; continue; }
            std::vector<MeshTriangle> built;
            for (const MeshTriangle& t : mit->second) built.push_back(mesh_triangle_build(t, in.xf, in.xf_inv));
            IdxInst* ex = nullptr; for (IdxInst& k : tri_index) if (k.handle == in.handle) ex = &k;
            if (ex && (ex->e - ex->s) == built.size()) {
                for (size_t i = 0; i < built.size(); i++) {   // triangles.rs:128-155
                    triangle_serialize(built[i], &gpu_triangles[9 * (ex->s + i)]);
                    BvhPrimitive& p = bvh_all[ex->s + i];
                    p.material_id = material_id; p.center = triangle_center(built[i]);
                    p.bounds = BBox(); for (int k = 0; k < 3; k++) p.bounds.add(built[i].positions[k]);
                }
            } else {
                if (ex) triangles_remove(in.handle);
                triangles_create(in.handle, built, material_id);
            }
        }
        return true;
    }
    // Engine::tick (lib.rs:301-395)
    void tick() {
        bool any_material_modified = dirty_materials; dirty_materials = false;
        bool any_image_modified = dirty_images; dirty_images = false;
        if (any_material_modified || any_image_modified) {  // materials.rs:79-85, material.rs:29-50
            gpu_materials.clear();
            for (const HostMaterial& m : materials) {
                Material g; g.base_color = m.base_color; g.base_color_texture = image_lookup(m.has_tex[0], m.tex[0]); g.emissive = m.emissive; g.emissive_texture = image_lookup(m.has_tex[1], m.tex[1]);
                g.roughness = pow_(m.perceptual_roughness, 2.0f); g.metallic = m.metallic; g.reflectance = m.reflectance; g.ior = m.ior;
                g.metallic_roughness_texture = image_lookup(m.has_tex[2], m.tex[2]); g.normal_map_texture = image_lookup(m.has_tex[3], m.tex[3]);
                gpu_materials.push_back(g);
            }
        }
        if (instances_refresh()) {  // bvh.rs:48-70
            bvh.run(bvh_all);
            std::vector<uint8_t> alpha; for (const HostMaterial& m : materials) alpha.push_back(m.alpha_blend ? 1 : 0);
            gpu_bvh.clear(); bvh_depth = 0;
            bvh.serialize(gpu_bvh, alpha, 0, 1, &bvh_depth);
        }
        // per-instance motion for the velocity map (passes/prim_raster.rs:198-223): curr_xform_inv + prev_transform
        tri_instance.assign(gpu_triangles.size() / 9, 0u);
        instance_xforms.assign(6 * std::max<size_t>(instances.size(), 1), v4z());
        for (size_t k = 0; k < instances.size(); k++) {
            const Inst& in = instances[k];
            const Affine* a[2] = {&in.xf_inv, &in.prev_xf};
            for (int j = 0; j < 2; j++) {
                instance_xforms[6 * k + 3 * j + 0] = v4(a[j]->x, a[j]->t.x);
                instance_xforms[6 * k + 3 * j + 1] = v4(a[j]->y, a[j]->t.y);
                instance_xforms[6 * k + 3 * j + 2] = v4(a[j]->z, a[j]->t.z);
            }
            for (const IdxInst& r : tri_index) if (r.handle == in.handle) for (size_t t = r.s; t < r.e; t++) tri_instance[t] = (u32)k;
        }
        world.light_count = next_light_id; world.sun_azimuth = sun_azimuth; world.sun_altitude = sun_altitude;
        if (dirty_sun) {  // lights.rs:84-99
            dirty_sun = false;
            V3 color = atm_transmittance_eval(atm_view_pos(), world_sun_dir(world));
            color = color * ATM_EXPOSURE * 5.0f;
            V3 sun_pos = world_sun_dir(world) * 1000.0f;
            light_update(0, UINT64_MAX, make_sun(sun_pos, color));
        }
        lights_flush();
        for (Cam* c : cameras) if (c->alive) c->frame = frame;   // camera_controller.rs:81-85
        frame += 1;
    }
    int create_camera(const HostCamera& hc) {  // camera_controller.rs:24-43
        Cam* c = new Cam(); c->cam = hc; c->st.init(hc.w, hc.h); c->frame = 0; c->alive = true;
        c->st.curr_camera = camera_serialize(hc.transform, hc.projection, hc.w, hc.h);
        c->st.prev_camera = c->st.curr_camera;
        cameras.push_back(c); return (int)cameras.size() - 1;
    }
    void update_camera(int h, const HostCamera& hc) {  // camera_controller.rs:45-63
        Cam* c = cameras[h];
        bool inval = c->cam.mode != hc.mode || c->cam.denoise != hc.denoise || c->cam.ref_depth != hc.ref_depth || c->cam.w != hc.w || c->cam.h != hc.h;
        c->cam = hc;
        c->st.prev_camera = c->st.curr_camera;
        c->st.curr_camera = camera_serialize(hc.transform, hc.projection, hc.w, hc.h);
        if (inval) { Camera a = c->st.curr_camera, b = c->st.prev_camera; c->st.init(hc.w, hc.h); c->st.curr_camera = a; c->st.prev_camera = b; }
    }
    Scene scene() {
        Scene sc; sc.triangles = gpu_triangles.data(); sc.bvh = gpu_bvh.data(); sc.bvh_len = gpu_bvh.size(); sc.materials = gpu_materials.data(); sc.lights = gpu_lights.data();
        sc.world = world; sc.blue_noise = blue_noise.data();
        sc.transmittance_lut.w = 256; sc.transmittance_lut.h = 64; sc.transmittance_lut.texels = luts.transmittance.data();
        sc.sky_lut.w = 256; sc.sky_lut.h = 256; sc.sky_lut.texels = luts.sky.data();
        sc.atlas = atlas.empty() ? nullptr : atlas.data(); sc.srgb_lut = srgb_lut.data();
        sc.tri_instance = tri_instance.data(); sc.instance_xforms = instance_xforms.data();
        return sc;
    }
    void run_atmosphere() {  // passes/atmosphere.rs:67-111
        if (!luts.have_static) { atm_generate_transmittance(luts.transmittance); atm_generate_scattering(luts.transmittance, luts.scattering); luts.have_static = true; }
        if (!luts.have_sky || luts.sky_altitude != sun_altitude) { atm_generate_sky(luts.transmittance, luts.scattering, world.sun_altitude, luts.sky); luts.sky_altitude = sun_altitude; luts.have_sky = true; }
    }
    // CameraController::render (camera_controller.rs:87-174) as an explicit step list: (pass id, work).  The ids are the device's
    // PassId values and the list is the device's schedule with strict arithmetic and one launch per reference dispatch
    // (ST_OPT_FUSED_PASSES = 0; K20 for both signals is one step, like the device's default fused reproject launch), so that a test
    // can stop between two passes (render_range) and read a pass's inputs before it overwrites them.
    struct Step { int pass; std::function<void()> run; };
    enum { S_PRIM_GBUFFER = 0, S_DI_SPATIAL_TRACE = 4, S_DI_RESOLVING = 6, S_GI_REPROJECTION = 7, S_GI_SPATIAL_TRACE = 12, S_GI_RESOLVING = 15,
           S_FRAME_REPROJECTION = 16, S_DENOISE_REPROJECT = 17, S_DENOISE_VARIANCE = 18, S_DENOISE_WAVELET = 19, S_COMPOSITION = 20,
           S_REF_TRACING = 21, S_REF_SHADING = 22, S_BVH_HEATMAP = 23 };
    std::vector<Step> schedule(int h) {
        Cam* c = cameras[h]; CamState* csp = &c->st; u32 f = c->frame; bool alt = (f % 2) == 1;
        const HostCamera hc = c->cam;
        Scene sc = scene();
        std::vector<Step> out;
        auto add = [&](int pass, std::function<void()> fn) { out.push_back(Step{pass, std::move(fn)}); };
        auto seed = [&](u32 k) { return dispatch_seed(seed_base, f, k); };
        if (hc.mode == MODE_BVH_HEATMAP) {
            add(S_BVH_HEATMAP, [=] { pass_bvh_heatmap(*csp, sc); });
            add(S_COMPOSITION, [=] { pass_frame_composition(*csp, alt, 5, false, false); });
            return out;
        }
        if (hc.mode == MODE_REFERENCE) {
            for (u32 d = 0; d <= hc.ref_depth; d++) {
                u32 sd = seed(D_REF_SHADING + d);
                add(S_REF_TRACING, [=] { pass_ref_tracing(*csp, sc, d); });
                add(S_REF_SHADING, [=] { pass_ref_shading(*csp, sc, sd, d); });
            }
            u32 sd = seed(D_REF_SHADING + 31);
            add(S_REF_SHADING, [=] { pass_ref_shading(*csp, sc, sd, 255); });
            add(S_COMPOSITION, [=] { pass_frame_composition(*csp, alt, 6, false, false); });
            return out;
        }
        bool needs_di = hc.mode == MODE_IMAGE || hc.mode == MODE_DI_DIFFUSE || hc.mode == MODE_DI_SPECULAR;
        bool needs_gi = hc.mode == MODE_IMAGE || hc.mode == MODE_GI_DIFFUSE || hc.mode == MODE_GI_SPECULAR;
        add(S_PRIM_GBUFFER, [=] { pass_prim_gbuffer(*csp, sc, alt); });
        if (!instances.empty()) {
            add(S_FRAME_REPROJECTION, [=] { pass_frame_reprojection(*csp, alt); });
            if (needs_di) {
                u32 s1 = seed(D_DI_SAMPLING), s2 = seed(D_DI_TEMPORAL), s3 = seed(D_DI_SPATIAL_PICK), s5 = seed(D_DI_SPATIAL_SAMPLE);
                add(D_DI_SAMPLING, [=] { pass_di_sampling(*csp, sc, alt, s1, f); });
                add(D_DI_TEMPORAL, [=] { pass_di_temporal(*csp, sc, alt, s2); });
                add(D_DI_SPATIAL_PICK, [=] { pass_di_spatial_pick(*csp, sc, alt, s3, f); });
                add(S_DI_SPATIAL_TRACE, [=] { pass_spatial_trace(*csp, sc, csp->di_diff_samples, csp->di_diff_curr_colors, csp->di_diff_stash); });
                add(D_DI_SPATIAL_SAMPLE, [=] { pass_di_spatial_sample(*csp, s5, f); });
                add(S_DI_RESOLVING, [=] { pass_di_resolving(*csp, sc, alt); });
            }
            if (needs_gi) {
                u32 sa = seed(D_GI_SAMPLING_A), sb = seed(D_GI_SAMPLING_B), st = seed(D_GI_TEMPORAL), sp = seed(D_GI_SPATIAL_PICK), ss = seed(D_GI_SPATIAL_SAMPLE);
                u32 ps = seed(D_GI_PREVIEW);   // both preview passes share one seed (passes/gi_preview_resampling.rs:58)
                u32 source;
                add(S_GI_REPROJECTION, [=] { pass_gi_reprojection(*csp, alt); });
                auto sampling = [&] {
                    add(D_GI_SAMPLING_A, [=] { pass_gi_sampling_a(*csp, sc, alt, sa, f); });
                    add(D_GI_SAMPLING_B, [=] { pass_gi_sampling_b(*csp, sc, alt, sb, f); });
                };
                if (frame_is_gi_tracing(f)) {
                    if (f % 2 == 0) sampling();
                    add(D_GI_TEMPORAL, [=] { pass_gi_temporal(*csp, alt, st, f); });
                    if (f % 2 == 1) {
                        add(D_GI_SPATIAL_PICK, [=] { pass_gi_spatial_pick(*csp, alt, sp, f); });
                        add(S_GI_SPATIAL_TRACE, [=] { pass_spatial_trace(*csp, sc, csp->gi_d0, csp->gi_d1, csp->gi_d2); });
                        add(D_GI_SPATIAL_SAMPLE, [=] { pass_gi_spatial_sample(*csp, ss, f); });
                        source = 1;
                    } else source = 0;
                } else {
                    sampling();
                    add(D_GI_TEMPORAL, [=] { pass_gi_temporal(*csp, alt, st, f); });
                    source = 0;
                }
                add(D_GI_PREVIEW, [=] { pass_gi_preview(*csp, alt, ps, source, 0, csp->gi_reservoirs[1], csp->gi_reservoirs[2], csp->gi_reservoirs[3]); });
                add(D_GI_PREVIEW, [=] { pass_gi_preview(*csp, alt, ps, 1, 1, csp->gi_reservoirs[1], csp->gi_reservoirs[3], csp->gi_reservoirs[0]); });
                add(S_GI_RESOLVING, [=] { pass_gi_resolving(*csp, alt, source); });
            }
        }
        if (hc.denoise) {  // passes/frame_denoising.rs:143-190
            int cur = alt ? 1 : 0, prv = alt ? 0 : 1;
            add(S_DENOISE_REPROJECT, [=] {
                CamState& cs = *csp;
                pass_denoise_reproject(cs, alt, cs.di_diff_prev_colors, cs.di_diff_moments[prv], cs.di_diff_samples, cs.di_diff_curr_colors, cs.di_diff_moments[cur]);
                pass_denoise_reproject(cs, alt, cs.gi_diff_prev_colors, cs.gi_diff_moments[prv], cs.gi_diff_samples, cs.gi_diff_curr_colors, cs.gi_diff_moments[cur]);
            });
            add(S_DENOISE_VARIANCE, [=] { pass_denoise_estimate_variance(*csp, alt); });
            for (u32 nth = 0; nth < 5; nth++) {
                add(S_DENOISE_WAVELET, [=] {
                    CamState& cs = *csp;
                    Buf* di_io[5][2] = {{&cs.di_diff_stash, &cs.di_diff_prev_colors}, {&cs.di_diff_prev_colors, &cs.di_diff_stash}, {&cs.di_diff_stash, &cs.di_diff_curr_colors},
                                        {&cs.di_diff_curr_colors, &cs.di_diff_stash}, {&cs.di_diff_stash, &cs.di_diff_curr_colors}};
                    Buf* gi_io[5][2] = {{&cs.gi_diff_stash, &cs.gi_diff_prev_colors}, {&cs.gi_diff_prev_colors, &cs.gi_diff_stash}, {&cs.gi_diff_stash, &cs.gi_diff_curr_colors},
                                        {&cs.gi_diff_curr_colors, &cs.gi_diff_stash}, {&cs.gi_diff_stash, &cs.gi_diff_curr_colors}};
                    pass_denoise_wavelet(cs, sc, alt, f, 1u << nth, (float)(1 + nth), *di_io[nth][0], *di_io[nth][1], *gi_io[nth][0], *gi_io[nth][1]);
                });
            }
        }
        bool den_di = hc.denoise && (hc.mode == MODE_IMAGE || hc.mode == MODE_DI_DIFFUSE);
        bool den_gi = hc.denoise && (hc.mode == MODE_IMAGE || hc.mode == MODE_GI_DIFFUSE);
        u32 mode = (u32)hc.mode;
        add(S_COMPOSITION, [=] { pass_frame_composition(*csp, alt, mode, den_di, den_gi); });
        return out;
    }
    // steps [first, last] of this frame's schedule (last < 0: to the end)
    void render_range(int h, int first, int last) {
        run_atmosphere();
        std::vector<Step> steps = schedule(h);
        if (last < 0 || last >= (int)steps.size()) last = (int)steps.size() - 1;
        for (int i = std::max(first, 0); i <= last; i++) steps[i].run();
    }
    void render_camera(int h) { render_range(h, 0, -1); }
};

}  // namespace orc
