// strolle_b200 — device library: rays + BVH traversal, triangles, G-buffer,
// camera, noise, BRDFs, lights, atmosphere sampling, reservoirs, MIS.
// CUDA counterparts of the strolle-gpu crate (reference file:line per item).
#pragma once
#include "st_math.cuh"
#include "st_types.h"

namespace ST_NS {
#if defined(ST_FAST) && ST_FAST
using namespace st;   // the POD layouts of st_types.h
#endif

#define ST_BVH_STACK 24          // strolle-gpu/src/lib.rs:76
#define ST_BLOCK 128             // threads per CTA for all per-pixel kernels (16 x 8 pixel tile)
// rows of a neighbouring strip that a gathering pass reads (strip partition, SURVEY §8e)
#define ST_REACH_SPATIAL 128     // ReSTIR spatial taps (di_spatial_resampling.rs:55-56, gi_spatial_resampling.rs, gi_preview_resampling.rs pass 1)
#define ST_REACH_PREVIEW2 64     // gi_preview_resampling.rs:64-70, pass 2
#define ST_REACH_SVGF 38         // K21 (3 rows) + the five K22 iterations (1 + 2 + 4 + 9 + 19 = 35) recomputed on the receiving side

ST_DEV float4 ldg4(const float4* p) { return __ldg(p); }
// Reservoir entries are 32 B (DI) / 64 B (GI), 32-byte aligned: a 32-byte aligned access touches exactly one sector (sm_90a issues it as
// two 128-bit accesses), so the scattered reservoir gathers fetch no half-used sectors and the mirrored stores to a neighbouring GPU are
// full 32-byte sectors on NVLink.
struct __align__(32) F8 { float4 a, b; };
ST_DEV F8 ld8(const float4* p) { return *reinterpret_cast<const F8*>(p); }
ST_DEV void st8(float4* p, float4 a, float4 b) { F8 v; v.a = a; v.b = b; *reinterpret_cast<F8*>(p) = v; }

// ---- Normal (strolle-gpu/src/normal.rs:9-34) --------------------------------
ST_DEV float2 oct_encode(float3 n) {
    n = n / (fabs_(n.x) + fabs_(n.y) + fabs_(n.z));
    float2 r;
    if (n.z >= 0.0f) r = f2(n.x, n.y);
    else r = f2(cpsign(1.0f - fabs_(n.y), n.x), cpsign(1.0f - fabs_(n.x), n.y));
    return r * 0.5f + f2(0.5f, 0.5f);
}
ST_DEV float3 oct_decode(float2 e) {
    float2 m = e * 2.0f - f2(1.0f, 1.0f);
    float3 n = f3(m.x, m.y, 1.0f - fabs_(m.x) - fabs_(m.y));
    float t = rmax(-n.z, 0.0f);
    n.x -= cpsign(t, n.x);
    n.y -= cpsign(t, n.y);
    return norm(n);
}

// ---- Ray (strolle-gpu/src/ray.rs) --------------------------------------------
struct Ray { float3 o, d, inv; float len; };
ST_DEV Ray ray_zero() { Ray r; r.o = f3s(0.f); r.d = f3s(0.f); r.inv = f3s(0.f); r.len = 0.f; return r; }
ST_DEV Ray ray_make(float3 o, float3 d) { Ray r; r.o = o; r.d = d; r.inv = f3(xdiv(1.0f, d.x), xdiv(1.0f, d.y), xdiv(1.0f, d.z)); r.len = kF32Max; return r; }   // ray.rs:22-30
ST_DEV Ray ray_make(float3 o, float3 d, float len) { Ray r = ray_make(o, d); r.len = len; return r; }
ST_DEV float3 ray_at(const Ray& r, float t) { return r.o + r.d * t; }
ST_DEV float ray_sphere(const Ray& r, float radius) {   // ray.rs:304-322
    float b = dot(r.o, r.d);
    float c = dot(r.o, r.o) - radius * radius;
    if (c > 0.0f && b > 0.0f) return -1.0f;
    float discr = b * b - c;
    if (discr < 0.0f) return -1.0f;
    else if (discr > b * b) return -b + sqrtf(discr);
    else return -b - sqrtf(discr);
}

// bu, bv, inv_det: the Möller–Trumbore barycentrics and 1 / determinant of the closest hit (normal mapping reads them; set by
// trace_closest only)
struct TriHit { float t; float3 point, normal; float2 uv; u32 material_id, triangle_id; float bu, bv, inv_det; };
ST_DEV TriHit trihit_none() { TriHit h; h.t = kF32Max; h.point = f3s(0.f); h.normal = f3s(0.f); h.uv = f2(0.f, 0.f); h.material_id = 0u; h.triangle_id = 0xffffffffu; return h; }
ST_DEV bool trihit_some(const TriHit& h) { return h.t < kF32Max; }
ST_DEV void trihit_pack(const TriHit& h, float4* d0, float4* d1) {   // hit.rs:112-120
    *d0 = f4(h.point, bitsf(h.material_id));
    float2 n = oct_encode(h.normal);
    *d1 = f4(n.x, n.y, h.uv.x, h.uv.y);
}
ST_DEV TriHit trihit_unpack(float4 d0, float4 d1) {   // hit.rs:95-110
    if (d0.x == 0.0f && d0.y == 0.0f && d0.z == 0.0f) return trihit_none();
    TriHit h; h.t = 0.0f; h.point = xyz(d0); h.normal = oct_decode(f2(d1.x, d1.y)); h.uv = f2(d1.z, d1.w); h.material_id = fbits(d0.w); h.triangle_id = 0xffffffffu;
    return h;
}

// slab test (ray.rs:273-302); fminf/fmaxf are NaN-ignoring like Rust's f32::min/max and only
// ordering of the result is consumed here, so the hardware min/max is used.
ST_DEV float box_entry(const Ray& r, float3 bmin, float3 bmax) {
    float t1x = xmul(xsub(bmin.x, r.o.x), r.inv.x), t2x = xmul(xsub(bmax.x, r.o.x), r.inv.x);
    float t1y = xmul(xsub(bmin.y, r.o.y), r.inv.y), t2y = xmul(xsub(bmax.y, r.o.y), r.inv.y);
    float t1z = xmul(xsub(bmin.z, r.o.z), r.inv.z), t2z = xmul(xsub(bmax.z, r.o.z), r.inv.z);
    float tmin = fmaxf(0.0f, fminf(t1x, t2x)), tmax = fminf(kF32Max, fmaxf(t1x, t2x));
    tmin = fmaxf(tmin, fminf(t1y, t2y)); tmax = fminf(tmax, fmaxf(t1y, t2y));
    tmin = fmaxf(tmin, fminf(t1z, t2z)); tmax = fminf(tmax, fmaxf(t1z, t2z));
    return (tmin <= tmax) ? tmin : kF32Max;
}

// Möller–Trumbore, two-sided (strolle-gpu/src/triangle.rs:64-113).  Only the three position
// float4s are fetched for the test; normals/uvs are loaded on acceptance.
ST_DEV bool tri_test(const float4* __restrict__ tri, const Ray& ray, float best, float* t_out, float* u_out, float* v_out, float* inv_det_out) {
    float4 a0 = ldg4(tri), a3 = ldg4(tri + 3), a6 = ldg4(tri + 6);
    float3 p0 = xyz(a0);
    float3 e1 = xsub3(xyz(a3), p0), e2 = xsub3(xyz(a6), p0);
    float3 pvec = xcross(ray.d, e2);
    float det = xdot(e1, pvec);
    if (fabs_(det) < kF32Eps) return false;
    float3 tvec = xsub3(ray.o, p0);
    float un = xdot(tvec, pvec);
    float3 qvec = xcross(tvec, e1);
    float vn = xdot(ray.d, qvec);
    float inv_det = xdiv(1.0f, det);
    float u = xmul(un, inv_det);
    float v = xmul(vn, inv_det);
    float t = xmul(xdot(e2, qvec), inv_det);
    if ((u < 0.0f) | (u > 1.0f) | (v < 0.0f) | (xadd(u, v) > 1.0f) | (t <= 0.0f) | (t >= best)) return false;
    *t_out = t; *u_out = u; *v_out = v; *inv_det_out = inv_det;
    return true;
}
ST_DEV void tri_shade(const float4* __restrict__ tri, float u, float v, float inv_det, float3* normal, float2* uv) {
    float4 a0 = ldg4(tri), a1 = ldg4(tri + 1), a3 = ldg4(tri + 3), a4 = ldg4(tri + 4), a6 = ldg4(tri + 6), a7 = ldg4(tri + 7);
    float3 n = xadd3(xadd3(xscale(xyz(a4), u), xscale(xyz(a7), v)), xscale(xyz(a1), xsub(xsub(1.0f, u), v)));
    *normal = xscale(xnorm(n), cpsign(1.0f, inv_det));
    float2 uv0 = f2(a0.w, a1.w), uv1 = f2(a3.w, a4.w), uv2 = f2(a6.w, a7.w);
    *uv = f2(xadd(xadd(uv0.x, xmul(xsub(uv1.x, uv0.x), u)), xmul(xsub(uv2.x, uv0.x), v)), xadd(xadd(uv0.y, xmul(xsub(uv1.y, uv0.y), u)), xmul(xsub(uv2.y, uv0.y), v)));
}

// Material::sample_atlas (strolle-gpu/src/material.rs:76-104): repeat-wrap the hit uv, map it into the
// image's atlas rect, nearest-texel fetch (wgpu default sampler, clamp-to-edge), sRGB decode of r,g,b.
ST_DEV float wrap_uv(float t) { return (t > 0.0f) ? fmodf(t, 1.0f) : xsub(1.0f, fmodf(-t, 1.0f)); }
ST_DEV uchar4 atlas_texel(const SceneDev& sc, float2 uv) {   // the nearest texel's bytes; the caller checks sc.atlas
    int x = to_i32_sat(floorf(xmul(uv.x, (float)kAtlasSize))), y = to_i32_sat(floorf(xmul(uv.y, (float)kAtlasSize)));
    x = max(0, min(x, (int)kAtlasSize - 1)); y = max(0, min(y, (int)kAtlasSize - 1));
    return __ldg(sc.atlas + (size_t)y * kAtlasSize + (size_t)x);
}
ST_DEV float2 atlas_uv(float2 hit_uv, float4 texture) {
    return f2(xadd(texture.x, xmul(wrap_uv(hit_uv.x), texture.z)), xadd(texture.y, xmul(wrap_uv(hit_uv.y), texture.w)));
}
ST_DEV float4 atlas_fetch(const SceneDev& sc, float2 uv) {
    if (!sc.atlas) return f4zero();
    uchar4 t = atlas_texel(sc, uv);
    return f4(__ldg(sc.srgb_lut + t.x), __ldg(sc.srgb_lut + t.y), __ldg(sc.srgb_lut + t.z), xdiv((float)t.w, 255.0f));
}
ST_DEV float4 sample_atlas(const SceneDev& sc, float2 hit_uv, float4 multiplier, float4 texture) {
    if (all_zero(texture)) return multiplier;
    float4 t = atlas_fetch(sc, atlas_uv(hit_uv, texture));
    return f4(xmul(multiplier.x, t.x), xmul(multiplier.y, t.y), xmul(multiplier.z, t.z), xmul(multiplier.w, t.w));
}
ST_DEV float4 mat_base_color(const SceneDev& sc, const GpuMaterial& m, float2 uv) { return sample_atlas(sc, uv, m.base_color, m.base_color_texture); }
ST_DEV float3 mat_emissive(const SceneDev& sc, const GpuMaterial& m, float2 uv) { return xyz(sample_atlas(sc, uv, m.emissive, m.emissive_texture)); }
ST_DEV float2 mat_metallic_roughness(const SceneDev& sc, const GpuMaterial& m, float2 uv) {   // material.rs:44-58
    float4 t = sample_atlas(sc, uv, f4(1.0f, m.roughness, m.metallic, 1.0f), m.metallic_roughness_texture);
    return f2(t.z, t.y);
}
// alpha of base_color at `uv` for the alpha test of Blend materials (ray.rs:212-229): reads only what it needs
ST_DEV float mat_alpha(const SceneDev& sc, u32 material_id, float2 uv) {
    const float4* m = reinterpret_cast<const float4*>(sc.materials + material_id);
    float4 base = ldg4(m), tex = ldg4(m + 1);
    return sample_atlas(sc, uv, base, tex).w;
}
// Normal mapping (ST_OPT_NORMAL_MAPS; DESIGN.md §2 "Normal maps"): the formula the reference keeps commented out in
// strolle-gpu/src/material.rs:105-140, with Bevy's back-face convention and a fallback to the interpolated normal.
//   N = tri_shade's normal before its sign flip, T4 = barycentric mix of the baked tangents (not renormalised), B = T4.w (N x T),
//   Nt = 2 texel / 255 - 1 (linear: a normal map is data, not colour), n' = normalize((Nt.x T + Nt.y B) + Nt.z N),
//   n' = N where n' is not finite or n'.N <= 0 (meshes without tangents bake NaN tangents), then the sign of inv_det.
// Explicit round-to-nearest operations only, so that the strict and the fast-shading builds give the same bits.
// `nmap` is the material's normal_map_texture rect; nothing beyond it is read for materials without a map.
ST_DEV float3 nmap_normal(const SceneDev& sc, const TriHit& h, float4 nmap) {
    if (all_zero(nmap) || !sc.atlas) return h.normal;
    const float s = cpsign(1.0f, h.inv_det);
    const float3 n = xscale(h.normal, s);   // exact: the factor is +-1
    const float4* tri = sc.triangles + 9u * (size_t)h.triangle_id;
    const float4 t0 = ldg4(tri + 2), t1 = ldg4(tri + 5), t2 = ldg4(tri + 8);
    const float u = h.bu, v = h.bv, w = xsub(xsub(1.0f, u), v);
    // same evaluation order as tri_shade's normal: (t1 u + t2 v) + t0 (1 - u - v)
    const float3 t = xadd3(xadd3(xscale(xyz(t1), u), xscale(xyz(t2), v)), xscale(xyz(t0), w));
    const float tw = xadd(xadd(xmul(t1.w, u), xmul(t2.w, v)), xmul(t0.w, w));
    const float3 b = xscale(xcross(n, t), tw);
    const uchar4 c = atlas_texel(sc, atlas_uv(h.uv, nmap));
    const float nx = xsub(xmul(2.0f, xdiv((float)c.x, 255.0f)), 1.0f), ny = xsub(xmul(2.0f, xdiv((float)c.y, 255.0f)), 1.0f),
                nz = xsub(xmul(2.0f, xdiv((float)c.z, 255.0f)), 1.0f);
    const float3 m = xnorm(xadd3(xadd3(xscale(t, nx), xscale(b, ny)), xscale(n, nz)));
    const bool ok = isfinite(m.x) && isfinite(m.y) && isfinite(m.z) && xdot(m, n) > 0.0f;
    return xscale(ok ? m : n, s);
}

// Per-thread traversal stack: a column of a CTA-shared array, stack[level * ST_BLOCK + tid]
// (bank = tid % 32 -> conflict-free), mirroring the reference's workgroup-shared stack
// (strolle-gpu/src/lib.rs:66-76).
struct TraceStack { u32* base; };
ST_DEV void stk_push(const TraceStack& s, u32 level, u32 v) { if (level < ST_BVH_STACK) s.base[level * ST_BLOCK] = v; }
ST_DEV u32 stk_get(const TraceStack& s, u32 level) { return s.base[level * ST_BLOCK]; }

// Ray::traverse, closest hit (ray.rs:114-266, Tracing::ReturnClosest).  Same visiting order as the
// reference (near child first, far child pushed iff far_d < best), hence the same winner on ties.
// one red.global per warp per traced ray batch, only when the host asked for ray statistics
ST_DEV void count_ray(const SceneDev& sc) {
    if (sc.ray_counter) {
        unsigned m = __activemask();
        if ((threadIdx.x & 31u) == (unsigned)(__ffs(m) - 1)) atomicAdd(sc.ray_counter, (unsigned long long)__popc(m));
    }
}
// takes a ray back out of the statistics: the primary rays a strip traces for rows it does not own (recomputed halo rows) are not work
// the frame asked for, and would flatter the strip-parallel Mrays/s
ST_DEV void uncount_ray(const SceneDev& sc) {
    if (sc.ray_counter) {
        unsigned m = __activemask();
        if ((threadIdx.x & 31u) == (unsigned)(__ffs(m) - 1)) atomicAdd(sc.ray_counter, 0ull - (unsigned long long)__popc(m));
    }
}
// Both traversals are written "while-while": a lane first walks internal nodes until it stands on a leaf entry (or runs out of
// work), then the whole run of leaf entries, then pops.  Per lane this is exactly the node sequence of the reference's single
// loop; across a warp it lets lanes that are still descending catch up before anyone starts triangle tests, so the expensive
// Möller–Trumbore code runs with more lanes active.
template <bool COUNT_MEMORY = false>
ST_DEV TriHit trace_closest(const Ray& ray, const SceneDev& sc, const TraceStack& stk, u32* used_memory = nullptr) {
    count_ray(sc);
    TriHit hit = trihit_none();
    if (sc.bvh_len == 0u) { if (COUNT_MEMORY && used_memory) *used_memory = 0u; return hit; }   // empty scene (no instance alive)
    float hu = 0.f, hv = 0.f, hid = 0.f;
    u32 ptr = 0u, sp = 0u, used = 0u;
    bool alive = true;
    while (alive) {
        float4 d0;
        for (;;) {   // descend: internal nodes
            if (COUNT_MEMORY) used += 16u;
            d0 = ldg4(sc.bvh + ptr);
            if (fbits(d0.w) != 0u) break;
            if (COUNT_MEMORY) used += 48u;
            float4 d1 = ldg4(sc.bvh + ptr + 1), d2 = ldg4(sc.bvh + ptr + 2), d3 = ldg4(sc.bvh + ptr + 3);
            u32 near_ptr = ptr + 4u, far_ptr = fbits(d1.w);
            float near_d = box_entry(ray, xyz(d0), xyz(d1));
            float far_d = box_entry(ray, xyz(d2), xyz(d3));
            if (far_d < near_d) { u32 tp = near_ptr; near_ptr = far_ptr; far_ptr = tp; float tf = near_d; near_d = far_d; far_d = tf; }
            if (far_d < hit.t) { stk_push(stk, sp, far_ptr); sp += 1u; }
            if (near_d < hit.t) { ptr = near_ptr; continue; }
            if (sp > 0u) { sp -= 1u; ptr = stk_get(stk, sp); continue; }
            alive = false; break;
        }
        if (!alive) break;
        for (;;) {   // the run of leaf entries that starts here (one float4 each, flag bit 0 = another follows)
            if (COUNT_MEMORY) used += 144u;
            u32 flags = fbits(d0.x), tid = fbits(d0.y), mid = fbits(d0.z);
            float t, u, v, inv_det;
            if (tri_test(sc.triangles + 9u * (size_t)tid, ray, hit.t, &t, &u, &v, &inv_det)) {
                bool accept = true;
                if (flags & 2u) {   // AlphaMode::Blend: the hit only counts where the base colour is opaque (ray.rs:212-229)
                    if (COUNT_MEMORY) used += 128u;   // size_of::<Material>() + one atlas texel (ray.rs:213-214)
                    float3 n_; float2 uv_;
                    tri_shade(sc.triangles + 9u * (size_t)tid, u, v, inv_det, &n_, &uv_);
                    accept = !(mat_alpha(sc, mid, uv_) < 1.0f);
                }
                if (accept) { hit.t = t; hu = u; hv = v; hid = inv_det; hit.triangle_id = tid; hit.material_id = mid; }
            }
            if (!(flags & 1u)) break;
            ptr += 1u;
            if (COUNT_MEMORY) used += 16u;
            d0 = ldg4(sc.bvh + ptr);
        }
        if (sp > 0u) { sp -= 1u; ptr = stk_get(stk, sp); }
        else alive = false;
    }
    if (trihit_some(hit)) {
        tri_shade(sc.triangles + 9u * (size_t)hit.triangle_id, hu, hv, hid, &hit.normal, &hit.uv);
        hit.point = ray_at(ray, hit.t);
        hit.bu = hu; hit.bv = hv; hit.inv_det = hid;
    }
    if (COUNT_MEMORY && used_memory) *used_memory = used;
    return hit;
}
// Ray::intersect, any hit (ray.rs:84-112, Tracing::ReturnFirst): true iff some triangle has 0 < t < len.
// The answer does not depend on visiting order; the reference's order is kept anyway.
ST_DEV bool trace_any(const Ray& ray, const SceneDev& sc, const TraceStack& stk) {
    count_ray(sc);
    if (sc.bvh_len == 0u) return false;
    const float best = ray.len;
    u32 ptr = 0u, sp = 0u;
    bool found = false, alive = true;
    while (alive) {
        float4 d0;
        for (;;) {
            d0 = ldg4(sc.bvh + ptr);
            if (fbits(d0.w) != 0u) break;
            float4 d1 = ldg4(sc.bvh + ptr + 1), d2 = ldg4(sc.bvh + ptr + 2), d3 = ldg4(sc.bvh + ptr + 3);
            u32 near_ptr = ptr + 4u, far_ptr = fbits(d1.w);
            float near_d = box_entry(ray, xyz(d0), xyz(d1));
            float far_d = box_entry(ray, xyz(d2), xyz(d3));
            if (far_d < near_d) { u32 tp = near_ptr; near_ptr = far_ptr; far_ptr = tp; float tf = near_d; near_d = far_d; far_d = tf; }
            if (far_d < best) { stk_push(stk, sp, far_ptr); sp += 1u; }
            if (near_d < best) { ptr = near_ptr; continue; }
            if (sp > 0u) { sp -= 1u; ptr = stk_get(stk, sp); continue; }
            alive = false; break;
        }
        if (!alive) break;
        for (;;) {
            float t, u, v, inv_det;
            if (tri_test(sc.triangles + 9u * (size_t)fbits(d0.y), ray, best, &t, &u, &v, &inv_det)) {
                if (!(fbits(d0.x) & 2u)) { found = true; break; }
                float3 n_; float2 uv_;
                tri_shade(sc.triangles + 9u * (size_t)fbits(d0.y), u, v, inv_det, &n_, &uv_);
                if (!(mat_alpha(sc, fbits(d0.z), uv_) < 1.0f)) { found = true; break; }
            }
            if (!(fbits(d0.x) & 1u)) break;
            ptr += 1u;
            d0 = ldg4(sc.bvh + ptr);
        }
        if (found) break;
        if (sp > 0u) { sp -= 1u; ptr = stk_get(stk, sp); }
        else alive = false;
    }
    return found;
}

// ---- G-buffer entry (strolle-gpu/src/gbuffer.rs:19-112) ------------------------
struct GBuf { float4 base_color; float3 normal; float metallic; float3 emissive; float roughness, reflectance, depth; };
ST_DEV GBuf gbuf_zero() { GBuf g; g.base_color = f4zero(); g.normal = f3s(0.f); g.metallic = 0.f; g.emissive = f3s(0.f); g.roughness = 0.f; g.reflectance = 0.f; g.depth = 0.f; return g; }
// Exact same values as the arithmetic form: the four base-colour channels are bytes, so
// pow(b / 255, 2.2) (and pow(a / 63, 2.2)) come from a 2 x 256-entry table built on the device with pow_det.
ST_DEV GBuf gbuf_unpack(const SceneDev& sc, float4 d0, float4 d1) {
    GBuf g;
    g.depth = d0.x;
    g.normal = oct_decode(f2(d0.y, d0.z));
    u32 b = fbits(d0.w);
    g.metallic = (float)(b & 0xffu) / 255.0f;
    g.roughness = sq((float)((b >> 8) & 0xffu) / 255.0f);
    g.reflectance = (float)((b >> 16) & 0xffu) / 255.0f;
    g.emissive = xyz(d1);
    u32 c = fbits(d1.w);
    g.base_color = f4(__ldg(sc.unpack_lut + (c & 0xffu)), __ldg(sc.unpack_lut + ((c >> 8) & 0xffu)), __ldg(sc.unpack_lut + ((c >> 16) & 0xffu)),
                      __ldg(sc.unpack_lut + 256u + ((c >> 24) & 0xffu)));
    return g;
}
ST_DEV GBuf gbuf_unpack(float4 d0, float4 d1) {
    GBuf g;
    g.depth = d0.x;
    g.normal = oct_decode(f2(d0.y, d0.z));
    u32 b = fbits(d0.w);
    g.metallic = (float)(b & 0xffu) / 255.0f;
    g.roughness = sq((float)((b >> 8) & 0xffu) / 255.0f);
    g.reflectance = (float)((b >> 16) & 0xffu) / 255.0f;
    g.emissive = xyz(d1);
    u32 c = fbits(d1.w);
    g.base_color = f4(pow_det((float)(c & 0xffu) / 255.0f, 2.2f), pow_det((float)((c >> 8) & 0xffu) / 255.0f, 2.2f),
                      pow_det((float)((c >> 16) & 0xffu) / 255.0f, 2.2f), pow_det((float)((c >> 24) & 0xffu) / 63.0f, 2.2f));
    return g;
}
ST_DEV void gbuf_pack(const GBuf& g, float4* d0, float4* d1) {
    float2 n = oct_encode(g.normal);
    u32 m = to_u32_sat(rclamp(g.metallic, 0.0f, 1.0f) * 255.0f);
    u32 r = to_u32_sat(rclamp(sqrtf(g.roughness), 0.0f, 1.0f) * 255.0f);
    u32 f = to_u32_sat(rclamp(g.reflectance, 0.0f, 1.0f) * 255.0f);
    *d0 = f4(g.depth, n.x, n.y, bitsf(pack_bytes(m, r, f, 1u)));
    const float ig = 1.0f / 2.2f;
    u32 cx = to_u32_sat(rclamp(pow_det(g.base_color.x, ig), 0.0f, 1.0f) * 255.0f);
    u32 cy = to_u32_sat(rclamp(pow_det(g.base_color.y, ig), 0.0f, 1.0f) * 255.0f);
    u32 cz = to_u32_sat(rclamp(pow_det(g.base_color.z, ig), 0.0f, 1.0f) * 255.0f);
    u32 cw = to_u32_sat(rclamp(pow_det(g.base_color.w, ig), 0.0f, 1.0f) * 63.0f);
    *d1 = f4(g.emissive.x, g.emissive.y, g.emissive.z, bitsf(pack_bytes(cx, cy, cz, cw)));
}
ST_DEV u32 gbuf_pack_color(float4 base_color) {
    const float ig = 1.0f / 2.2f;
    u32 cx = to_u32_sat(rclamp(pow_det(base_color.x, ig), 0.0f, 1.0f) * 255.0f);
    u32 cy = to_u32_sat(rclamp(pow_det(base_color.y, ig), 0.0f, 1.0f) * 255.0f);
    u32 cz = to_u32_sat(rclamp(pow_det(base_color.z, ig), 0.0f, 1.0f) * 255.0f);
    u32 cw = to_u32_sat(rclamp(pow_det(base_color.w, ig), 0.0f, 1.0f) * 63.0f);
    return pack_bytes(cx, cy, cz, cw);
}
// gbuf_pack with the colour bytes already packed (per-material table for untextured materials)
ST_DEV void gbuf_pack_pre(const GBuf& g, u32 color_bits, float4* d0, float4* d1) {
    float2 n = oct_encode(g.normal);
    u32 m = to_u32_sat(rclamp(g.metallic, 0.0f, 1.0f) * 255.0f);
    u32 r = to_u32_sat(rclamp(sqrtf(g.roughness), 0.0f, 1.0f) * 255.0f);
    u32 f = to_u32_sat(rclamp(g.reflectance, 0.0f, 1.0f) * 255.0f);
    *d0 = f4(g.depth, n.x, n.y, bitsf(pack_bytes(m, r, f, 1u)));
    *d1 = f4(g.emissive.x, g.emissive.y, g.emissive.z, bitsf(color_bits));
}
ST_DEV float gbuf_clamped_roughness(const GBuf& g) { return rclamp(g.roughness, 0.089f * 0.089f, 1.0f); }

// ---- Camera (strolle-gpu/src/camera.rs) ------------------------------------------
ST_DEV const Mat4& cam_pv(const GpuCamera& c) { return *reinterpret_cast<const Mat4*>(c.projection_view); }
ST_DEV const Mat4& cam_n2w(const GpuCamera& c) { return *reinterpret_cast<const Mat4*>(c.ndc_to_world); }
ST_DEV float2 cam_clip_to_screen(const GpuCamera& c, float4 pos) {
    float2 ndc = f2(pos.x, pos.y) / pos.w;
    ndc = f2(ndc.x, -ndc.y);
    return (0.5f * ndc + f2(0.5f, 0.5f)) * f2(c.screen.x, c.screen.y);
}
ST_DEV float2 cam_world_to_screen(const GpuCamera& c, float3 p) { return cam_clip_to_screen(c, mat_mul(cam_pv(c), f4(p, 1.0f))); }
ST_DEV bool cam_contains_i(const GpuCamera& c, int x, int y) { return x >= 0 && y >= 0 && x < to_i32_sat(c.screen.x) && y < to_i32_sat(c.screen.y); }
ST_DEV bool cam_contains_u(const GpuCamera& c, u32 x, u32 y) { return x < to_u32_sat(c.screen.x) && y < to_u32_sat(c.screen.y); }
ST_DEV bool cam_contains_f(const GpuCamera& c, float2 p) { return p.x >= 0.0f && p.y >= 0.0f && p.x < c.screen.x && p.y < c.screen.y; }
ST_DEV uint2 cam_contain(const GpuCamera& c, int x, int y) {   // camera.rs:57-77, wrapping i32
    int sx = to_i32_sat(c.screen.x), sy = to_i32_sat(c.screen.y);
    if (x < 0) x = (int)(0u - (u32)x);
    if (y < 0) y = (int)(0u - (u32)y);
    if (x >= sx) x = (int)((u32)sx - (u32)x + (u32)sx - 1u);
    if (y >= sy) y = (int)((u32)sy - (u32)y + (u32)sy - 1u);
    return make_uint2((u32)x, (u32)y);
}
ST_DEV Ray cam_ray(const GpuCamera& c, u32 px, u32 py) {   // camera.rs:80-93
    float2 size = f2(c.screen.x, c.screen.y);
    float2 p = f2((float)px, (float)py) + f2(0.5f, 0.5f);
    float2 ndc = p * 2.0f / size - f2(1.0f, 1.0f);
    ndc = f2(ndc.x, -ndc.y);
    float3 far_plane = project_point(cam_n2w(c), f3(ndc.x, ndc.y, kF32Eps));
    float3 near_plane = project_point(cam_n2w(c), f3(ndc.x, ndc.y, 1.0f));
    return ray_make(near_plane, norm(far_plane - near_plane));
}
ST_DEV bool cam_is_eq(const GpuCamera& a, const GpuCamera& b) {   // camera.rs:103-106
    const float* p = reinterpret_cast<const float*>(a.projection_view);
    const float* q = reinterpret_cast<const float*>(b.projection_view);
    bool ok = true;
    for (int i = 0; i < 16; i++) ok = ok && (fabs_(p[i] - q[i]) <= 0.0025f);
    return ok;
}

// ---- Texture filtering (ST_OPT_TEXTURE_FILTER; DESIGN.md §2 "Texture filtering") ------------------------------------------------
// The level of detail, the texel addresses and the weights use the x*() primitives only, so the filtered value is the same in the
// strict and the fast-shading builds.
// log2 of a finite x > 0: the exponent bits plus the Cephes logf polynomial of the mantissa, times log2(e) (st_device_math op 7)
ST_DEV float log2_x(float x) {
    u32 bits = fbits(x);
    int e;
    if ((bits & 0x7f800000u) == 0u) { x = xmul(x, 8388608.0f); bits = fbits(x); e = (int)((bits >> 23) & 0xffu) - 126 - 23; }
    else e = (int)((bits >> 23) & 0xffu) - 126;
    float m = bitsf((bits & 0x007fffffu) | 0x3f000000u);   // [0.5, 1)
    if (m < 0.707106781186547524f) { e -= 1; m = xsub(xadd(m, m), 1.0f); } else m = xsub(m, 1.0f);
    const float z = xmul(m, m);
    float y = 7.0376836292e-2f;
    y = xadd(xmul(y, m), -1.1514610310e-1f); y = xadd(xmul(y, m), 1.1676998740e-1f); y = xadd(xmul(y, m), -1.2420140846e-1f);
    y = xadd(xmul(y, m), 1.4249322787e-1f); y = xadd(xmul(y, m), -1.6668057665e-1f); y = xadd(xmul(y, m), 2.0000714765e-1f);
    y = xadd(xmul(y, m), -2.4999993993e-1f); y = xadd(xmul(y, m), 3.3333331174e-1f);
    y = xmul(xmul(y, m), z);
    y = xadd(y, xmul(-0.5f, z));
    const float ln_m = xadd(m, y);   // ln(1 + m), m in [sqrt(1/2) - 1, sqrt(2) - 1)
    return xadd(xmul(ln_m, 1.44269504088896341f), (float)e);
}
ST_DEV float xlen(float3 a) { return xsqrt(xdot(a, a)); }
ST_DEV float4 xscale4(float4 a, float s) { return f4(xmul(a.x, s), xmul(a.y, s), xmul(a.z, s), xmul(a.w, s)); }
ST_DEV float4 xadd4(float4 a, float4 b) { return f4(xadd(a.x, b.x), xadd(a.y, b.y), xadd(a.z, b.z), xadd(a.w, b.w)); }
// cam_ray through the x*() primitives (the same bits as cam_ray in the strict build)
ST_DEV void cam_ray_x(const GpuCamera& c, u32 px, u32 py, float3* o, float3* d) {
    const Mat4& m = cam_n2w(c);
    const float nx = xsub(xdiv(xmul(xadd((float)px, 0.5f), 2.0f), c.screen.x), 1.0f);
    const float ny = -xsub(xdiv(xmul(xadd((float)py, 0.5f), 2.0f), c.screen.y), 1.0f);
    float3 pl[2];
    const float zs[2] = {kF32Eps, 1.0f};
#pragma unroll
    for (int k = 0; k < 2; k++) {
        float4 r = xscale4(m.c[0], nx);
        r = xadd4(r, xscale4(m.c[1], ny)); r = xadd4(r, xscale4(m.c[2], zs[k])); r = xadd4(r, m.c[3]);
        const float rw = xdiv(1.0f, r.w);
        pl[k] = f3(xmul(r.x, rw), xmul(r.y, rw), xmul(r.z, rw));
    }
    *o = pl[1]; *d = xnorm(xsub3(pl[0], pl[1]));
}
// Ray-cone width at a hit `t` along the ray.  (o0, d0), (o1, d1), (o2, d2): the camera rays of pixel (px, py), (px + 1, py) and
// (px, py + 1).  Primary hits: max(|(o1 - o0) + t (d1 - d0)|, |(o2 - o0) + t (d2 - d0)|) (perspective and orthographic alike).
// Secondary hits start a fresh cone at the segment's origin: t max(|d1 - d0|, |d2 - d0|).
ST_DEV float texf_cone_width(const GpuCamera& c, u32 px, u32 py, float t, bool primary) {
    float3 o0, d0, o1, d1, o2, d2;
    cam_ray_x(c, px, py, &o0, &d0); cam_ray_x(c, px + 1u, py, &o1, &d1); cam_ray_x(c, px, py + 1u, &o2, &d2);
    if (primary) return rmax(xlen(xadd3(xsub3(o1, o0), xscale(xsub3(d1, d0), t))), xlen(xadd3(xsub3(o2, o0), xscale(xsub3(d2, d0), t))));
    return xmul(t, rmax(xlen(xsub3(d1, d0)), xlen(xsub3(d2, d0))));
}
// What the filtered fetch needs of a hit: its triangle, the ray direction and the cone width there
struct TexFoot { u32 tri; float3 dir; float w; };
// lambda = 0.5 log2(q), q = A_uv W H w^2 |c| / (c.d)^2, c = (p1 - p0) x (p2 - p0), A_uv = |(uv1 - uv0) x (uv2 - uv0)|, clamped to
// [0, levels - 1]; q <= 0 or NaN -> 0, q = +inf -> the last level
ST_DEV float texf_lambda(const SceneDev& sc, const TexFoot& f, u32 W, u32 H, u32 levels) {
    const float4* tri = sc.triangles + 9u * (size_t)f.tri;
    const float4 a0 = ldg4(tri), a1 = ldg4(tri + 1), a3 = ldg4(tri + 3), a4 = ldg4(tri + 4), a6 = ldg4(tri + 6), a7 = ldg4(tri + 7);
    const float3 p0 = xyz(a0);
    const float3 c = xcross(xsub3(xyz(a3), p0), xsub3(xyz(a6), p0));
    const float auv = fabs_(xsub(xmul(xsub(a3.w, a0.w), xsub(a7.w, a1.w)), xmul(xsub(a6.w, a0.w), xsub(a4.w, a1.w))));
    const float cd = xdot(c, f.dir);
    const float q = xdiv(xmul(xmul(xmul(xmul(auv, (float)W), (float)H), xmul(f.w, f.w)), xlen(c)), xmul(cd, cd));
    const float top = (float)(levels - 1u);
    if (!(q > 0.0f)) return 0.0f;
    if (q == finf()) return top;
    return rclamp(xmul(0.5f, log2_x(q)), 0.0f, top);
}
// Bilinear on level k of an image (level 0: its atlas rect at (ax, ay), W x H; level 1 at pool texel `off1`): s = u w_k - 0.5,
// taps floor(s) and floor(s) + 1 modulo w_k (the same for v), rgb decoded through the sRGB table, alpha / 255
ST_DEV float4 texf_texel(const SceneDev& sc, const uchar4* src, size_t i) {
    const uchar4 t = __ldg(src + i);
    return f4(__ldg(sc.srgb_lut + t.x), __ldg(sc.srgb_lut + t.y), __ldg(sc.srgb_lut + t.z), xdiv((float)t.w, 255.0f));
}
ST_DEV float4 xlerp4(float4 a, float4 b, float wa, float wb) {
    return f4(xadd(xmul(a.x, wa), xmul(b.x, wb)), xadd(xmul(a.y, wa), xmul(b.y, wb)), xadd(xmul(a.z, wa), xmul(b.z, wb)), xadd(xmul(a.w, wa), xmul(b.w, wb)));
}
ST_DEV float4 texf_bilinear(const SceneDev& sc, const TexFilterDev& tf, u32 ax, u32 ay, u32 W, u32 H, u32 off1, u32 k, float u, float v) {
    u32 w = W, h = H, off = off1;
    for (u32 j = 1u; j <= k; j++) { if (j > 1u) off += w * h; w = max(1u, w >> 1); h = max(1u, h >> 1); }
    const float s = xsub(xmul(u, (float)w), 0.5f), t = xsub(xmul(v, (float)h), 0.5f);
    const float sx = floorf(s), sy = floorf(t);
    const float fx = xsub(s, sx), fy = xsub(t, sy);
    const int ix = max(-1, min(to_i32_sat(sx), (int)w - 1)), iy = max(-1, min(to_i32_sat(sy), (int)h - 1));
    const u32 xa = ix < 0 ? w - 1u : (u32)ix, xb = (u32)(ix + 1) >= w ? 0u : (u32)(ix + 1);
    const u32 ya = iy < 0 ? h - 1u : (u32)iy, yb = (u32)(iy + 1) >= h ? 0u : (u32)(iy + 1);
    const uchar4* src; size_t stride;
    if (k == 0u) { src = sc.atlas + (size_t)ay * kAtlasSize + ax; stride = kAtlasSize; } else { src = tf.pool + off; stride = w; }
    const float4 c00 = texf_texel(sc, src, ya * stride + xa), c10 = texf_texel(sc, src, ya * stride + xb);
    const float4 c01 = texf_texel(sc, src, yb * stride + xa), c11 = texf_texel(sc, src, yb * stride + xb);
    const float gx = xsub(1.0f, fx), gy = xsub(1.0f, fy);
    return xlerp4(xlerp4(c00, c10, gx, fx), xlerp4(c01, c11, gx, fx), gy, fy);
}
// Material::sample_atlas with the filter: trilinear between levels floor(lambda) and floor(lambda) + 1, times the factor.  `slot`:
// 0 base colour, 1 emissive, 2 metallic-roughness.
ST_DEV float4 texf_sample(const SceneDev& sc, const TexFilterDev& tf, u32 material_id, u32 slot, float4 rect, float4 multiplier, float2 hit_uv, const TexFoot& f) {
    if (all_zero(rect) || !sc.atlas) return sample_atlas(sc, hit_uv, multiplier, rect);
    const uint2 e = __ldg(tf.table + 3u * (size_t)material_id + slot);
    const u32 levels = max(e.y, 1u);
    const u32 ax = to_u32_sat(xmul(rect.x, (float)kAtlasSize)), ay = to_u32_sat(xmul(rect.y, (float)kAtlasSize));
    const u32 W = to_u32_sat(xmul(rect.z, (float)kAtlasSize)), H = to_u32_sat(xmul(rect.w, (float)kAtlasSize));
    const float u = wrap_uv(hit_uv.x), v = wrap_uv(hit_uv.y);
    const float lambda = levels > 1u ? texf_lambda(sc, f, W, H, levels) : 0.0f;
    const float lf = floorf(lambda);
    const u32 k0 = (u32)lf;
    const float fl = xsub(lambda, lf);
    float4 t = texf_bilinear(sc, tf, ax, ay, W, H, e.x, k0, u, v);
    if (fl > 0.0f && k0 + 1u < levels) t = xlerp4(t, texf_bilinear(sc, tf, ax, ay, W, H, e.x, k0 + 1u, u, v), xsub(1.0f, fl), fl);
    return f4(xmul(multiplier.x, t.x), xmul(multiplier.y, t.y), xmul(multiplier.z, t.z), xmul(multiplier.w, t.w));
}

// ---- Hit / Surface (hit.rs:8-73, surface.rs) -----------------------------------------
struct Hit { float3 origin, dir, point; GBuf g; };
ST_DEV Hit hit_zero() { Hit h; h.origin = f3s(0.f); h.dir = f3s(0.f); h.point = f3s(0.f); h.g = gbuf_zero(); return h; }
ST_DEV Hit hit_make(const Ray& ray, const GBuf& g) { Hit h; h.origin = ray.o; h.dir = ray.d; h.point = ray_at(ray, g.depth - 0.01f); h.g = g; return h; }
ST_DEV bool hit_some(const Hit& h) { return h.g.depth != 0.0f; }

struct Surf { float3 normal; float depth, roughness; };
ST_DEV Surf surf_decode(float4 d) { Surf s; s.normal = oct_decode(f2(d.x, d.y)); s.depth = d.z; s.roughness = d.w; return s; }
ST_DEV float surf_similarity(const Surf& self, const Surf& other) {   // surface.rs:21-47
    if (self.depth == 0.0f || other.depth == 0.0f) return 0.0f;
    float d = rmax(dot(self.normal, other.normal), 0.0f);
    float ns = (d <= 0.5f) ? 0.0f : 2.0f * d;
    float t = fabs_(self.depth - other.depth);
    float ds = (t >= 0.1f * other.depth) ? 0.0f : 1.0f;
    return ns * ds;
}

// ---- Reprojection + bilinear history fetch (reprojection.rs, utils/bilinear_filter.rs) -----
struct Reproj { float px, py, confidence; u32 validity; };
ST_DEV Reproj reproj_decode(float4 d) { Reproj r; r.px = d.x; r.py = d.y; r.confidence = d.z; r.validity = fbits(d.w); return r; }
ST_DEV float4 reproj_encode(const Reproj& r) { return f4(r.px, r.py, r.confidence, bitsf(r.validity)); }
ST_DEV bool reproj_some(const Reproj& r) { return r.confidence > 0.0f; }
ST_DEV uint2 reproj_round(const Reproj& r) { return make_uint2(to_u32_sat(roundf(r.px)), to_u32_sat(roundf(r.py))); }
ST_DEV bool reproj_exact(const Reproj& r) { float2 f = f2(r.px - floorf(r.px), r.py - floorf(r.py)); return len2(f) == 0.0f; }
ST_DEV float4 history_fetch(const Reproj& r, const float4* __restrict__ tex, int w, int h) {
    if (reproj_exact(r)) {
        uint2 p = reproj_round(r);
        if ((int)p.x >= w || (int)p.y >= h) return f4zero();
        return tex[(size_t)p.y * w + p.x];
    }
    int x0 = to_i32_sat(floorf(r.px)), x1 = to_i32_sat(ceilf(r.px)), y0 = to_i32_sat(floorf(r.py)), y1 = to_i32_sat(ceilf(r.py));
    int xs[4] = {x0, x1, x0, x1}, ys[4] = {y0, y0, y1, y1};
    float4 s[4]; float wt[4];
#pragma unroll
    for (int i = 0; i < 4; i++) {
        s[i] = f4zero(); wt[i] = 0.0f;
        if ((r.validity & (1u << i)) > 0u && xs[i] >= 0 && ys[i] >= 0) {
            if (xs[i] < w && ys[i] < h) s[i] = tex[(size_t)ys[i] * w + xs[i]];
            wt[i] = 1.0f;
        }
    }
    float ux = r.px - truncf(r.px), uy = r.py - truncf(r.py);
    float4 wv = f4(wt[0], wt[1], wt[2], wt[3]) * f4((1.0f - ux) * (1.0f - uy), ux * (1.0f - uy), (1.0f - ux) * uy, ux * uy);
    float wsum = dot(wv, f4(1.f, 1.f, 1.f, 1.f));
    if (wsum == 0.0f) return f4zero();
    return (s[0] * wv.x + s[1] * wv.y + s[2] * wv.z + s[3] * wv.w) / wsum;
}

// ---- Noise (noise/white.rs, noise/blue.rs) ------------------------------------------------
struct Rng { u32 s; };
ST_DEV Rng rng_make(u32 seed, u32 x, u32 y) { Rng r; r.s = seed ^ (48619u * x) ^ (95461u * y); return r; }
ST_DEV u32 rng_u32(Rng& r) {
    r.s = r.s * 747796405u + 2891336453u;
    u32 word = ((r.s >> ((r.s >> 28) + 4u)) ^ r.s) * 277803737u;
    return (word >> 22) ^ word;
}
ST_DEV float rng_f(Rng& r) { return xmul((float)rng_u32(r), 2.3283064365386963e-10f); }   // / 2^32 (white.rs:44-46), exact as a product
ST_DEV float2 rng_disk(Rng& r) {
    float radius = sqrtf(rng_f(r));
    float a = rng_f(r) * kPi * 2.0f;
    float s, c; sincos_det(a, &s, &c);
    return f2(c, s) * radius;
}
ST_DEV float3 rng_sphere(Rng& r) {
    float phi = rng_f(r) * 2.0f * kPi;
    float cos_theta = rng_f(r) * 2.0f - 1.0f;
    float u = rng_f(r);
    float theta = acos_det(cos_theta);
    float rr = sqrtf(u);
    float st_, ct_, sp, cp; sincos_det(theta, &st_, &ct_); sincos_det(phi, &sp, &cp);
    return f3(rr * st_ * cp, rr * st_ * sp, rr * ct_);
}
ST_DEV float3 rng_hemisphere(Rng& r, float3 normal) {
    float cos_theta = rng_f(r);
    float sin_theta = sqrtf(1.0f - sq(cos_theta));
    float phi = 2.0f * kPi * rng_f(r);
    float3 t, b; ortho_pair(normal, &t, &b);
    float sp, cp; sincos_det(phi, &sp, &cp);
    return (t * cp + b * sp) * sin_theta + normal * cos_theta;
}
ST_DEV float4 blue_noise(const SceneDev& sc, u32 x, u32 y, u32 frame) {
    u32 ux = (x + 71u * frame) % 256u, uy = (y + 11u * frame) % 256u;
    uchar4 t = __ldg(sc.blue_noise + uy * 256u + ux);
    return f4((float)t.x / 255.0f, (float)t.y / 255.0f, (float)t.z / 255.0f, (float)t.w / 255.0f);
}

// ---- BRDFs (brdf.rs) ----------------------------------------------------------------------------
struct BrdfS { float3 dir; float pdf; float3 radiance; };
ST_DEV float3 brdf_diffuse(const GBuf& g) { return xyz(g.base_color) * (1.0f - g.metallic) / kPi; }
ST_DEV float ggx_d(float n_dot_h, float roughness) { float a2 = roughness * roughness; float d = (n_dot_h * a2 - n_dot_h) * n_dot_h + 1.0f; return a2 / (kPi * d * d); }
ST_DEV float ggx_g(float n_dot_l, float n_dot_v, float roughness) {
    float k = roughness * roughness / 2.0f;
    float gv = n_dot_v / (n_dot_v * (1.0f - k) + k);
    float gl = n_dot_l / (n_dot_l * (1.0f - k) + k);
    return gv * gl;
}
ST_DEV float3 brdf_specular(const GBuf& g, float3 l, float3 v) {   // brdf.rs:46-79
    if (g.metallic <= 0.0f) return f3s(0.f);
    float a = gbuf_clamped_roughness(g);
    float3 n = g.normal;
    float3 h = norm(l + v);
    float n_dot_l = sat(dot(n, l)), n_dot_h = sat(dot(n, h)), l_dot_h = sat(dot(l, h)), n_dot_v = sat(dot(n, v));
    if (n_dot_l <= 0.0f || n_dot_v <= 0.0f) return f3s(0.f);
    float d = ggx_d(n_dot_h, a);
    float gg = ggx_g(n_dot_l, n_dot_v, a);
    float3 f0 = f3s(0.16f * g.reflectance * g.reflectance * (1.0f - g.metallic)) + xyz(g.base_color) * g.metallic;
    float f90 = sat(dot(f0, f3s(50.0f * 0.33f)));
    float3 f = f0 + (f3s(f90) - f0) * pow_det(rmax(1.0f - l_dot_h, 0.001f), 5.0f);
    return d * gg * f / (4.0f * n_dot_l * n_dot_v);
}
ST_DEV BrdfS brdf_layered_sample(const GBuf& g, Rng& rng, float3 v) {   // brdf.rs:125-138 (+26-32, 82-113)
    BrdfS s;
    if (rng_f(rng) < g.metallic) {
        float r0 = rng_f(rng), r1 = rng_f(rng);
        float a = gbuf_clamped_roughness(g);
        float3 n = g.normal;
        float a2 = sq(a);
        float3 b, t; ortho_pair(n, &b, &t);
        float cos_theta = sqrtf(rmax(0.0f, (1.0f - r0) / ((a2 - 1.0f) * r0 + 1.0f)));
        float sin_theta = sqrtf(rmax(0.0f, 1.0f - cos_theta * cos_theta));
        float phi = r1 * kPi * 2.0f;
        float sp, cp; sincos_det(phi, &sp, &cp);
        float3 h = t * (sin_theta * cp) + b * (sin_theta * sp) + n * cos_theta;
        float n_dot_h = sat(dot(n, h)), h_dot_v = sat(dot(h, v));
        s.dir = norm(2.0f * h_dot_v * h - v);
        s.pdf = ggx_d(n_dot_h, a) * n_dot_h / (4.0f * h_dot_v);
        s.radiance = brdf_specular(g, s.dir, v);
        s.pdf /= g.metallic;
    } else {
        s.dir = rng_hemisphere(rng, g.normal);
        s.pdf = 1.0f / kPi;
        s.radiance = brdf_diffuse(g);
        s.pdf /= 1.0f - g.metallic;
    }
    return s;
}

// ---- Lights (light.rs) -----------------------------------------------------------------------------
struct LightRad { float3 radiance, diff, spec; };
ST_DEV LightRad lightrad_zero() { LightRad r; r.radiance = f3s(0.f); r.diff = f3s(0.f); r.spec = f3s(0.f); return r; }
ST_DEV float3 lightrad_sum(const LightRad& r) { return r.radiance * (r.diff + r.spec); }
ST_DEV GpuLight light_load(const SceneDev& sc, u32 id) {
    const float4* p = reinterpret_cast<const float4*>(sc.lights + id);
    GpuLight l; l.d0 = ldg4(p); l.d1 = ldg4(p + 1); l.d2 = ldg4(p + 2); l.d3 = ldg4(p + 3); l.prev_d0 = ldg4(p + 4); l.prev_d1 = ldg4(p + 5); l.prev_d2 = ldg4(p + 6);
    return l;
}
ST_DEV GpuLight light_prev(GpuLight l) { l.d0 = l.prev_d0; l.d1 = l.prev_d1; l.d2 = l.prev_d2; return l; }
ST_DEV bool light_is_none(const GpuLight& l) { return fbits(l.d2.x) == 0u; }
ST_DEV bool light_contains(const GpuLight& l, float3 p) { return dist(xyz(l.d0), p) <= l.d0.w; }
ST_DEV LightRad light_radiance(const GpuLight& self, const Hit& hit) {   // light.rs:143-207
    float3 l = xyz(self.d0) - hit.point;
    float f_angle;
    if (fbits(self.d2.x) == 1u) f_angle = 1.0f;
    else {
        float3 sd = oct_decode(f2(self.d2.y, self.d2.z));
        float3 hv = hit.point - xyz(self.d0);
        float angle = acos_approx_glam(dot(sd, hv) / sqrtf(len2(sd) * len2(hv)));   // Vec3::angle_between
        f_angle = sat(1.0f - pow_det(angle / self.d2.w, 3.0f));
    }
    float range = self.d1.w, f_dist;
    if (range == finf()) f_dist = 1.0f;
    else {
        float l2 = len2(l);
        float inv_r2 = 1.0f / sq(range);
        float factor = l2 * inv_r2;
        float smooth = sat(1.0f - factor * factor);
        float att = smooth * smooth;
        f_dist = att / rmax(l2, 0.0001f);
    }
    float f_cos = sat(dot(hit.g.normal, norm(l)));
    LightRad out;
    out.diff = brdf_diffuse(hit.g);
    {
        float3 v = -hit.dir;
        float3 n = hit.g.normal;
        float3 r = reflect3(-v, n);
        float3 c2r = dot(l, r) * r - l;
        float tt = self.d0.w * (1.0f / sqrtf(dot(c2r, c2r)));
        float3 closest = l + c2r * sat(tt);
        float inv_len = 1.0f / sqrtf(dot(closest, closest));
        float cr = gbuf_clamped_roughness(hit.g);
        float t2 = cr + self.d0.w * 0.5f * inv_len;
        float i_rough = cr / sat(t2);
        float intensity = sq(i_rough);
        float3 ll = closest * inv_len;
        out.spec = intensity * brdf_specular(hit.g, ll, v);
    }
    out.radiance = xyz(self.d1) * f_angle * f_dist * f_cos;
    return out;
}
ST_DEV Ray light_ray_wnoise(const GpuLight& self, Rng& rng, float3 hit_point) {   // light.rs:209-215
    float3 lp = xyz(self.d0) + self.d0.w * rng_sphere(rng);
    float3 l2h = hit_point - lp;
    return ray_make(lp, norm(l2h), len(l2h));
}
ST_DEV Ray light_ray_bnoise(const GpuLight& self, float2 sample, float3 hit_point) {   // light.rs:217-239
    float3 to_light = xyz(self.d0) - hit_point;
    float3 light_dir = norm(to_light);
    float light_distance = len(to_light);
    float light_radius = self.d0.w / light_distance;
    float3 tg, bt; ortho_pair(light_dir, &tg, &bt);
    float angle = 2.0f * kPi * sample.x;
    float radius = sqrtf(sample.y);
    float sa, ca; sincos_det(angle, &sa, &ca);
    float2 disk = f2(sa, ca) * radius * light_radius;
    float3 rd = light_dir + disk.x * tg + disk.y * bt;
    rd = norm(rd);
    return ray_make(hit_point + rd * light_distance, -rd, light_distance);
}

// ---- Atmosphere sampling (atmosphere.rs:86-205) --------------------------------------------------------
#define ST_ATM_GROUND 6.360f
#define ST_ATM_TOP 6.460f
ST_DEV float3 atm_view_pos() { return f3(0.0f, ST_ATM_GROUND + 0.0002f, 0.0f); }
// explicit f32 bilinear fetch, clamp-to-edge, texel centres at +0.5
ST_DEV float3 lut_fetch(const float4* __restrict__ lut, int w, int h, float2 uv) {
    float fx = uv.x * (float)w - 0.5f, fy = uv.y * (float)h - 0.5f;
    float x0f = floorf(fx), y0f = floorf(fy);
    float tx = fx - x0f, ty = fy - y0f;
    int x0 = to_i32_sat(x0f), y0 = to_i32_sat(y0f);
    int x1 = x0 + 1, y1 = y0 + 1;
    x0 = max(0, min(x0, w - 1)); x1 = max(0, min(x1, w - 1)); y0 = max(0, min(y0, h - 1)); y1 = max(0, min(y1, h - 1));
    float3 a = xyz(ldg4(lut + (size_t)y0 * w + x0)), b = xyz(ldg4(lut + (size_t)y0 * w + x1));
    float3 c = xyz(ldg4(lut + (size_t)y1 * w + x0)), d = xyz(ldg4(lut + (size_t)y1 * w + x1));
    float3 top = a + (b - a) * tx, bot = c + (d - c) * tx;
    return top + (bot - top) * ty;
}
ST_DEV float3 atm_lut(const float4* __restrict__ lut, int w, int h, float3 pos, float3 sun_dir) {   // atmosphere.rs:183-204
    float height = len(pos);
    float3 up = pos / height;
    float czen = dot(sun_dir, up);
    float u = sat(0.5f + 0.5f * czen);
    float v = sat((height - ST_ATM_GROUND) / (ST_ATM_TOP - ST_ATM_GROUND));
    return lut_fetch(lut, w, h, f2(u, v));
}
ST_DEV float3 world_sun_dir(const GpuWorld& w) {   // world.rs:19-25
    float sa, ca, sz, cz; sincos_det(w.sun_altitude, &sa, &ca); sincos_det(w.sun_azimuth, &sz, &cz);
    return f3(ca * sz, sa, -ca * cz);
}
ST_DEV float3 atmosphere_sample(const SceneDev& sc, float3 sun_dir, float3 ray_dir) {
    float3 vp = atm_view_pos();
    float height = len(vp);
    float3 up = vp / height;
    float horizon;
    { float t = sq(height) - sq(ST_ATM_GROUND); t = sqrtf(t) / height; horizon = acos_det(rclamp(t, -1.0f, 1.0f)); }
    float altitude = horizon - acos_det(dot(ray_dir, up));
    float azimuth;
    if (fabs_(altitude) > (0.5f * kPi - 0.0001f)) azimuth = 0.0f;
    else {
        float3 right = cross(sun_dir, up);
        float3 forward = cross(up, right);
        float3 proj = norm(ray_dir - up * dot(ray_dir, up));
        azimuth = atan2_det(dot(proj, right), dot(proj, forward)) + kPi;
    }
    float u = azimuth / (2.0f * kPi);
    float v = 0.5f + 0.5f * cpsign(sqrtf(fabs_(altitude) * 2.0f / kPi), altitude);
    float3 lum = lut_fetch(sc.sky_lut, 256, 256, f2(u, v));
    // sun disk + bloom (atmosphere.rs:148-172)
    const float sun_solid_angle = 0.53f * kPi / 180.0f;
    float min_cos = cos_det(sun_solid_angle);
    float cos_theta = dot(ray_dir, sun_dir);
    float3 sun_lum;
    if (cos_theta >= min_cos) sun_lum = f3s(1.0f);
    else {
        float offset = min_cos - cos_theta;
        float gaussian = exp_det(-offset * 50000.0f) * 0.5f;
        float inv_bloom = 1.0f / (0.02f + offset * 300.0f) * 0.01f;
        sun_lum = f3s(gaussian + inv_bloom);
    }
    {
        float3 t = clamp3((sun_lum - f3s(0.002f)) / (f3s(1.0f) - f3s(0.002f)), f3s(0.f), f3s(1.f));
        sun_lum = t * t * (f3s(3.0f) - 2.0f * t);
    }
    if (len2(sun_lum) > 0.0f) {
        Ray r = ray_make(vp, ray_dir);
        if (ray_sphere(r, ST_ATM_GROUND) >= 0.0f) sun_lum = f3s(0.f);
        else sun_lum = sun_lum * atm_lut(sc.transmittance_lut, 256, 64, vp, sun_dir);
    }
    lum = lum + sun_lum;
    lum = lum * 20.0f;
    return lum;
}

// ---- Environment map (st_set_environment_map; DESIGN.md §2 "Environment map") --------------------------------------------------
// The lookup uses the x*() primitives only, so the sky it gives is the same in the strict and the fast-shading builds.
// acos_det / atan2_det's Cephes kernels through the x*() primitives (st_device_math ops 8 and 9)
ST_DEV float asin_core_x(float x) {
    const float z = xmul(x, x);
    float p = 4.2163199048e-2f;
    p = xadd(xmul(p, z), 2.4181311049e-2f); p = xadd(xmul(p, z), 4.5470025998e-2f); p = xadd(xmul(p, z), 7.4953002686e-2f);
    p = xadd(xmul(p, z), 1.6666752422e-1f);
    return xadd(xmul(xmul(p, z), x), x);
}
ST_DEV float acos_x(float x) {
    if (!(x == x)) return x;
    if (x < -1.0f || x > 1.0f) return fnan();
    if (x > 0.5f) return xmul(2.0f, asin_core_x(xsqrt(xmul(0.5f, xsub(1.0f, x)))));
    if (x < -0.5f) return xsub(kPi, xmul(2.0f, asin_core_x(xsqrt(xmul(0.5f, xadd(1.0f, x))))));
    if (x >= 0.0f) return xsub(kHalfPi, asin_core_x(x));
    return xadd(kHalfPi, asin_core_x(-x));
}
ST_DEV float atan_core_x(float x) {   // x >= 0
    float y;
    if (x > 2.414213562373095f) { y = kHalfPi; x = -xdiv(1.0f, x); }
    else if (x > 0.4142135623730950f) { y = 0.7853981633974483f; x = xdiv(xsub(x, 1.0f), xadd(x, 1.0f)); }
    else y = 0.0f;
    const float z = xmul(x, x);
    float p = 8.05374449538e-2f;
    p = xsub(xmul(p, z), 1.38776856032e-1f); p = xadd(xmul(p, z), 1.99777106478e-1f); p = xsub(xmul(p, z), 3.33329491539e-1f);
    return xadd(y, xadd(xmul(xmul(p, z), x), x));
}
ST_DEV float atan2_x(float y, float x) {
    if (!(x == x) || !(y == y)) return fnan();
    if (y == 0.0f) {
        if (x > 0.0f || (x == 0.0f && !(fbits(x) >> 31))) return y;
        return cpsign(kPi, y);
    }
    if (x == 0.0f) return cpsign(kHalfPi, y);
    float a = atan_core_x(xdiv(fabs_(y), fabs_(x)));
    if (x < 0.0f) a = xsub(kPi, a);
    return cpsign(a, y);
}
// The map's radiance along d (as the pass has it, not renormalised): theta = acos(d.y), phi = atan2(d.x, -d.z); u = (phi + rotation)
// / 2 pi + 0.5, v = theta / pi; columns floor(u W - 0.5) and the next, wrapped modulo W, rows floor(v H - 0.5) and the next, clamped;
// blended as lut_fetch blends, times the intensity.  A non-finite u or v gives 0.
ST_DEV float3 env_sample(const EnvMapDev& em, float3 d) {
    const float theta = acos_x(rclamp(d.y, -1.0f, 1.0f)), phi = atan2_x(d.x, -d.z);
    const float u = xadd(xmul(xadd(phi, em.rotation), 0.15915494309189535f), 0.5f), v = xmul(theta, 0.3183098861837907f);
    if (!(fabs_(u) < finf()) || !(fabs_(v) < finf())) return f3s(0.0f);
    const float s = xsub(xmul(u, (float)em.w), 0.5f), t = xsub(xmul(v, (float)em.h), 0.5f);
    const float sx = floorf(s), sy = floorf(t);
    const float tx = xsub(s, sx), ty = xsub(t, sy);
    const int W = (int)em.w, H = (int)em.h;
    int x0 = to_i32_sat(sx) % W; if (x0 < 0) x0 += W;
    const int x1 = x0 + 1 == W ? 0 : x0 + 1;
    const int iy = to_i32_sat(sy);
    const int y0 = max(0, min(iy, H - 1)), y1 = max(0, min(iy + 1, H - 1));
    const float3 a = xyz(ldg4(em.texels + (size_t)y0 * W + x0)), b = xyz(ldg4(em.texels + (size_t)y0 * W + x1));
    const float3 c = xyz(ldg4(em.texels + (size_t)y1 * W + x0)), e = xyz(ldg4(em.texels + (size_t)y1 * W + x1));
    const float3 top = f3(xadd(a.x, xmul(xsub(b.x, a.x), tx)), xadd(a.y, xmul(xsub(b.y, a.y), tx)), xadd(a.z, xmul(xsub(b.z, a.z), tx)));
    const float3 bot = f3(xadd(c.x, xmul(xsub(e.x, c.x), tx)), xadd(c.y, xmul(xsub(e.y, c.y), tx)), xadd(c.z, xmul(xsub(e.z, c.z), tx)));
    const float3 r = f3(xadd(top.x, xmul(xsub(bot.x, top.x), ty)), xadd(top.y, xmul(xsub(bot.y, top.y), ty)), xadd(top.z, xmul(xsub(bot.z, top.z), ty)));
    return xscale(r, em.intensity);
}
// The sky radiance along `dir` at the four sites that evaluate it: the map when the ENVM instantiation runs, else atmosphere_sample
template <bool ENVM>
ST_DEV float3 sky_radiance(const SceneDev& sc, const EnvMapDev& em, float3 sun_dir, float3 dir) {
    return ENVM ? env_sample(em, dir) : atmosphere_sample(sc, sun_dir, dir);
}

// ---- Environment map sampling (ST_OPT_ENVIRONMENT_MAP_SAMPLING; DESIGN.md §2 "Environment map sampling") ------------------------
// The draw and its density use the x*() primitives only, as the lookup does, so both builds give the same bits.
// The strict build's sincos_det (Cephes, three-part pi/4 reduction) through the x*() primitives
ST_DEV void sincos_x(float xx, float* s_out, float* c_out) {
    float x = fabs_(xx);
    u32 j = to_u32_sat(xmul(1.27323954473516f, x));
    float y = (float)j;
    if (j & 1u) { j += 1u; y = xadd(y, 1.0f); }
    j &= 7u;
    x = xsub(xsub(xsub(x, xmul(y, 0.78515625f)), xmul(y, 2.4187564849853515625e-4f)), xmul(y, 3.77489497744594108e-8f));
    const float z = xmul(x, x);
    const float ps = xadd(xmul(xmul(xsub(xmul(xadd(xmul(-1.9515295891e-4f, z), 8.3321608736e-3f), z), 1.6666654611e-1f), z), x), x);
    const float pc = xadd(xsub(xmul(xmul(xadd(xmul(xsub(xmul(2.443315711809948e-5f, z), 1.388731625493765e-3f), z), 4.166664568298827e-2f), z), z),
                               xmul(0.5f, z)), 1.0f);
    float s = (j == 0u) ? ps : (j == 2u) ? pc : (j == 4u) ? -ps : -pc;
    const float c = (j == 0u) ? pc : (j == 2u) ? -ps : (j == 4u) ? -pc : ps;
    if (fbits(xx) & 0x80000000u) s = -s;
    *s_out = s; *c_out = c;
}
// The first index i < n with cdf[i] > t or cdf[i] == last (the second clause catches t == last, reached by a draw of exactly 1).
ST_DEV u32 env_cdf_find(const float* cdf, u32 n, float t, float last) {
    u32 lo = 0u, hi = n - 1u;
    while (lo < hi) {
        const u32 mid = (lo + hi) >> 1;
        const float c = __ldg(cdf + mid);
        if (c > t || c == last) hi = mid; else lo = mid + 1u;
    }
    return lo;
}
// A direction drawn with density env_pdf: the row from the marginal CDF at xi1 * total, the column from that row's conditional CDF
// at xi2 * (the row's last value), each offset inside its cell the remainder over the cell's CDF difference (below 1);
// u = (j + du) / W, v = (i + dv) / H, phi = (u - 0.5) 2 pi - rotation, theta = pi v, d = (sin theta sin phi, cos theta,
// -sin theta cos phi): the exact inverse of the lookup's theta = acos(d.y), phi = atan2(d.x, -d.z).
ST_DEV float3 env_draw(const EnvMapDev& em, float xi1, float xi2) {
    const u32 W = em.w, H = em.h;
    const float below_one = 0.99999994039535522f;   // the largest float below 1
    const float* M = em.cdf;
    const float t = xmul(xi1, em.total);
    const u32 i = env_cdf_find(M, H, t, em.total);
    const float m0 = i ? __ldg(M + i - 1u) : 0.0f, m1 = __ldg(M + i);
    const float dv = fminf(xdiv(xsub(t, m0), xsub(m1, m0)), below_one);
    const float* C = em.cdf + H + (size_t)i * W;
    const float rt = __ldg(C + W - 1u);
    const float t2 = xmul(xi2, rt);
    const u32 j = env_cdf_find(C, W, t2, rt);
    const float c0 = j ? __ldg(C + j - 1u) : 0.0f, c1 = __ldg(C + j);
    const float du = fminf(xdiv(xsub(t2, c0), xsub(c1, c0)), below_one);
    const float u = xdiv(xadd((float)j, du), (float)W), v = xdiv(xadd((float)i, dv), (float)H);
    const float phi = xsub(xmul(xsub(u, 0.5f), 6.283185307179586f), em.rotation), theta = xmul(kPi, v);
    float st, ct, sp, cp;
    sincos_x(theta, &st, &ct); sincos_x(phi, &sp, &cp);
    return f3(xmul(st, sp), ct, -xmul(st, cp));
}
// The solid-angle density of env_draw at d: u, v as env_sample computes them, the cell (floor(u W) wrapped, floor(v H) clamped),
// p = ((row's marginal CDF difference / total) (cell's conditional CDF difference / the row's last value)) (W H) / (2 pi^2 sin theta),
// sin theta = sqrt(max(0, 1 - d.y^2)); 0 where the cell cannot be drawn, +inf where sin theta = 0.
ST_DEV float env_pdf(const EnvMapDev& em, float3 d) {
    const float theta = acos_x(rclamp(d.y, -1.0f, 1.0f)), phi = atan2_x(d.x, -d.z);
    const float u = xadd(xmul(xadd(phi, em.rotation), 0.15915494309189535f), 0.5f), v = xmul(theta, 0.3183098861837907f);
    if (!(fabs_(u) < finf()) || !(fabs_(v) < finf())) return 0.0f;
    const int W = (int)em.w, H = (int)em.h;
    int j = to_i32_sat(floorf(xmul(u, (float)W))) % W; if (j < 0) j += W;
    const int i = max(0, min(to_i32_sat(floorf(xmul(v, (float)H))), H - 1));
    const float* M = em.cdf;
    const float* C = em.cdf + H + (size_t)i * W;
    const float pr = xsub(__ldg(M + i), i ? __ldg(M + i - 1) : 0.0f), pc = xsub(__ldg(C + j), j ? __ldg(C + j - 1) : 0.0f);
    if (!(pr > 0.0f) || !(pc > 0.0f)) return 0.0f;
    const float st = xsqrt(fmaxf(0.0f, xsub(1.0f, xmul(d.y, d.y))));
    if (st == 0.0f) return finf();
    const float prob = xmul(xdiv(pr, em.total), xdiv(pc, __ldg(C + W - 1)));
    return xdiv(xmul(prob, xmul((float)W, (float)H)), xmul(19.739208802178716f, st));
}
// K12's one-sample mixture (ENV_SAMPLED): q(w) / kappa(w) for a bounce direction w at a surface g seen along v.  q = 1/2 p_bsdf +
// 1/2 p_env with p_bsdf = (1 - m) / 2 pi [n.w > 0] + m p_ggx(w); kappa = (1 - m)^2 / 2 [n.w > 0] + m^2 [p_ggx(w) > 0] is what the
// reference's per-branch pdfs estimate; +inf where kappa = 0 (the candidate then carries w = 0).
ST_DEV float env_mixture_pdf(const EnvMapDev& em, const GBuf& g, float3 v, float3 w) {
    const float m = g.metallic;
    const float3 n = g.normal;
    const bool up = xdot(n, w) > 0.0f;
    float pg = 0.0f;
    if (m > 0.0f) {
        const float a = gbuf_clamped_roughness(g), a2 = xmul(a, a);
        const float3 h = xnorm(xadd3(w, v));
        const float n_dot_h = sat(xdot(n, h)), h_dot_v = sat(xdot(h, v));
        if (n_dot_h > 0.0f && h_dot_v > 0.0f) {
            const float dd = xadd(xmul(xsub(xmul(n_dot_h, a2), n_dot_h), n_dot_h), 1.0f);
            const float dist = xdiv(a2, xmul(xmul(kPi, dd), dd));
            pg = xdiv(xmul(dist, n_dot_h), xmul(4.0f, h_dot_v));
        }
    }
    const float om = xsub(1.0f, m);
    const float kappa = xadd(up ? xmul(xmul(om, om), 0.5f) : 0.0f, pg > 0.0f ? xmul(m, m) : 0.0f);
    if (!(kappa > 0.0f)) return finf();
    const float pb = xadd(up ? xmul(om, 0.15915494309189535f) : 0.0f, xmul(m, pg));
    const float q = xadd(xmul(0.5f, pb), xmul(0.5f, env_pdf(em, w)));
    return xdiv(q, kappa);
}

// ---- Reservoirs (reservoir.rs, reservoir/{di,gi,ephemeral,mis}.rs) ------------------------------------------
struct DiRes { float m, w; float pdf, confidence; u32 light_id; float3 light_point; bool occluded; };
ST_DEV DiRes di_zero() { DiRes r; r.m = 0.f; r.w = 0.f; r.pdf = 0.f; r.confidence = 0.f; r.light_id = 0u; r.light_point = f3s(0.f); r.occluded = false; return r; }
ST_DEV DiRes di_load(const float4* __restrict__ buf, size_t id) {   // di.rs:17-35
    F8 e = ld8(buf + 2 * id);
    float4 d0 = e.a, d1 = e.b;
    u32 b = fbits(d0.w);
    DiRes r; r.m = d0.x; r.w = d0.y; r.pdf = d0.z; r.confidence = (float)((b >> 8) & 0xffu); r.occluded = (b & 0xffu) > 0u;
    r.light_point = xyz(d1); r.light_id = fbits(d1.w);
    return r;
}
ST_DEV void di_store(const DiRes& r, float4* __restrict__ buf, size_t id) {   // di.rs:37-59
    st8(buf + 2 * id, f4(r.m, r.w, r.pdf, bitsf(pack_bytes(r.occluded ? 1u : 0u, to_u32_sat(r.confidence), 0u, 0u))), f4(r.light_point, bitsf(r.light_id)));
}
// ---- strip partition: a store that also lands in the neighbouring strips' copy when the row is within `reach` of an edge ----
ST_DEV void mirror4(const CameraDev& cam, float4* p, float4 v, u32 y, int reach) {
    if (cam.mirror_up != 0 && (int)y < cam.own_y0 + reach) *reinterpret_cast<float4*>(reinterpret_cast<char*>(p) + cam.mirror_up) = v;
    if (cam.mirror_dn != 0 && (int)y >= cam.own_y1 - reach) *reinterpret_cast<float4*>(reinterpret_cast<char*>(p) + cam.mirror_dn) = v;
}
ST_DEV void store4m(const CameraDev& cam, float4* p, float4 v, u32 y, int reach) { *p = v; mirror4(cam, p, v, y, reach); }
ST_DEV void store8m(const CameraDev& cam, float4* p, float4 a, float4 b, u32 y, int reach) {
    st8(p, a, b);
    if (cam.mirror_up != 0 && (int)y < cam.own_y0 + reach) st8(reinterpret_cast<float4*>(reinterpret_cast<char*>(p) + cam.mirror_up), a, b);
    if (cam.mirror_dn != 0 && (int)y >= cam.own_y1 - reach) st8(reinterpret_cast<float4*>(reinterpret_cast<char*>(p) + cam.mirror_dn), a, b);
}
ST_DEV void di_store_m(const CameraDev& cam, const DiRes& r, float4* __restrict__ buf, size_t id, u32 y, int reach) {
    store8m(cam, buf + 2 * id, f4(r.m, r.w, r.pdf, bitsf(pack_bytes(r.occluded ? 1u : 0u, to_u32_sat(r.confidence), 0u, 0u))), f4(r.light_point, bitsf(r.light_id)), y, reach);
}
// Reservoir::update specialised: copies sample fields of `s` into `dst` on acceptance (reservoir.rs:24-39)
ST_DEV bool di_update(DiRes& dst, Rng& rng, const DiRes& s, float weight) {
    dst.m += 1.0f; dst.w += weight;
    if (rng_f(rng) * dst.w < weight) { dst.pdf = s.pdf; dst.confidence = s.confidence; dst.light_id = s.light_id; dst.light_point = s.light_point; dst.occluded = s.occluded; return true; }
    return false;
}
ST_DEV float res_norm(float w, float pdf, float num, float den) { float d = pdf * den; return (d == 0.0f) ? 0.0f : (w * num) / d; }   // reservoir.rs:63-71
ST_DEV float di_pdf_with(const DiRes& s, const GpuLight& light, Hit hit) {   // di.rs:108-117
    hit.g.base_color = f4(1.f, 1.f, 1.f, 1.f);
    if (!light_is_none(light) && light_contains(light, s.light_point)) return luma(lightrad_sum(light_radiance(light, hit)));
    return 0.0f;
}
ST_DEV Ray di_ray(const DiRes& s, float3 hit_point) { float3 d = hit_point - s.light_point; return ray_make(s.light_point, norm(d), len(d)); }   // di.rs:119-123

struct GiRes { float m, w, confidence; float pdf; u32 rng; float3 radiance, v1, v2, v2n; };
ST_DEV GiRes gi_zero() { GiRes r; r.m = 0.f; r.w = 0.f; r.confidence = 0.f; r.pdf = 0.f; r.rng = 0u; r.radiance = f3s(0.f); r.v1 = f3s(0.f); r.v2 = f3s(0.f); r.v2n = f3s(0.f); return r; }
ST_DEV GiRes gi_load(const float4* __restrict__ buf, size_t id) {   // gi.rs:19-40
    F8 e0 = ld8(buf + 4 * id), e1 = ld8(buf + 4 * id + 2);
    float4 d0 = e0.a, d1 = e0.b, d2 = e1.a, d3 = e1.b;
    GiRes r; r.radiance = xyz(d0); r.m = d0.w; r.v1 = xyz(d1); r.w = d1.w; r.v2 = xyz(d2); r.pdf = d2.w;
    r.v2n = oct_decode(f2(d3.x, d3.y)); r.confidence = d3.z; r.rng = fbits(d3.w);
    return r;
}
ST_DEV void gi_store(const GiRes& r, float4* __restrict__ buf, size_t id) {   // gi.rs:42-57
    float2 n = oct_encode(r.v2n);
    st8(buf + 4 * id, f4(r.radiance, r.m), f4(r.v1, r.w));
    st8(buf + 4 * id + 2, f4(r.v2, r.pdf), f4(n.x, n.y, r.confidence, bitsf(r.rng)));
}
ST_DEV void gi_store_m(const CameraDev& cam, const GiRes& r, float4* __restrict__ buf, size_t id, u32 y, int reach) {
    float2 n = oct_encode(r.v2n);
    store8m(cam, buf + 4 * id, f4(r.radiance, r.m), f4(r.v1, r.w), y, reach);
    store8m(cam, buf + 4 * id + 2, f4(r.v2, r.pdf), f4(n.x, n.y, r.confidence, bitsf(r.rng)), y, reach);
}
ST_DEV void gi_take_sample(GiRes& dst, const GiRes& s) { dst.pdf = s.pdf; dst.rng = s.rng; dst.radiance = s.radiance; dst.v1 = s.v1; dst.v2 = s.v2; dst.v2n = s.v2n; }
ST_DEV bool gi_update(GiRes& dst, Rng& rng, const GiRes& s, float weight) {
    dst.m += 1.0f; dst.w += weight;
    if (rng_f(rng) * dst.w < weight) { gi_take_sample(dst, s); return true; }
    return false;
}
ST_DEV bool gi_merge(GiRes& dst, Rng& rng, const GiRes& s, float pdf) {   // reservoir.rs:41-53
    if (s.m <= 0.0f) return false;
    dst.m += s.m - 1.0f;
    return gi_update(dst, rng, s, s.w * s.m * pdf);
}
ST_DEV bool gi_exists(const GiRes& s) { return !(s.v2.x == 0.0f && s.v2.y == 0.0f && s.v2.z == 0.0f); }
ST_DEV float3 gi_dir(const GiRes& s, float3 p) { return norm(s.v2 - p); }
ST_DEV float gi_cosine(const GiRes& s, const Hit& hit) { return rmax(dot(gi_dir(s, hit.point), hit.g.normal), 0.0f); }
ST_DEV float3 gi_spec(const GiRes& s, const Hit& hit) { return brdf_specular(hit.g, gi_dir(s, hit.point), -hit.dir); }
ST_DEV float gi_pdf(const GiRes& s, Hit hit) {   // gi.rs:98-112
    if (!gi_exists(s)) return 0.0f;
    hit.g.base_color = f4(1.f, 1.f, 1.f, 1.f);
    float diff = luma(brdf_diffuse(hit.g));
    float spec = luma(gi_spec(s, hit));
    return luma(s.radiance) * gi_cosine(s, hit) * (diff + spec);
}
ST_DEV Ray gi_ray(const GiRes& s, float3 hit_point) { return ray_make(hit_point, gi_dir(s, hit_point), dist(s.v2, hit_point) - 0.01f); }   // gi.rs:114-117
ST_DEV void gi_partial_jac(const GiRes& s, float3 p, float* d, float* c) { float3 v = p - s.v2; *d = len(v); *c = sat(dot(s.v2n, v / *d)); }
ST_DEV float gi_jacobian(const GiRes& s, float3 new_point) {   // gi.rs:135-151
    if (!gi_exists(s)) return 1.0f;
    float nd, nc, od, oc;
    gi_partial_jac(s, new_point, &nd, &nc);
    gi_partial_jac(s, s.v1, &od, &oc);
    float x = nc * od * od, y = oc * nd * nd;
    return (y == 0.0f) ? 0.0f : x / y;
}

// EphemeralReservoir::build (ephemeral.rs:14-55): RIS over min(light_count, 16) uniformly drawn lights
struct EphRes { float m, w; u32 light_id; LightRad rad; };
ST_DEV EphRes ephemeral_build(Rng& rng, const SceneDev& sc, const Hit& hit) {
    EphRes res; res.m = 0.f; res.w = 0.f; res.light_id = 0u; res.rad = lightrad_zero();
    float res_pdf = 0.0f;
    u32 lc = sc.world.light_count;
    u32 max_samples = lc < 16u ? lc : 16u;
    float ipdf = (float)lc;
    for (u32 nth = 0u; nth < max_samples; nth++) {
        u32 id = rng_u32(rng) % lc;
        LightRad lr = light_radiance(light_load(sc, id), hit);
        float pdf = sqrtf(luma(lr.radiance));
        float weight = pdf * ipdf;
        res.m += 1.0f; res.w += weight;
        if (rng_f(rng) * res.w < weight) { res.light_id = id; res.rad = lr; res_pdf = pdf; }
    }
    res.w = res_norm(res.w, res_pdf, 1.0f, res.m);
    return res;
}

// ---- Light grid (ST_OPT_LIGHT_GRID; DESIGN.md §2 "Light grid") -----------------------------------------------------------
// A slot is cullable when its radiance is provably zero outside its range sphere: a point light (kind 1) with a finite position and
// colour and 2^-60 <= range <= 2^60 (|position| <= 2^60: no squared distance the test or light_radiance forms overflows or flushes).
// Spot lights stay in every list: their f_angle is NaN where the cone axis or the offset degenerates, and sat() keeps NaN.
ST_DEV bool lgrid_cullable(const GpuLight& l) {
    const float big = 1.152921504606846976e18f, tiny = 8.673617379884035472e-19f;   // 2^60, 2^-60
    if (fbits(l.d2.x) != 1u) return false;
    if (!(fabsf(l.d0.x) <= big && fabsf(l.d0.y) <= big && fabsf(l.d0.z) <= big)) return false;
    if (!(isfinite(l.d1.x) && isfinite(l.d1.y) && isfinite(l.d1.z))) return false;
    return l.d1.w >= tiny && l.d1.w <= big;
}
// The list a point samples from: `ids` = nullptr means every slot (identity), as with the option off.
struct LgList { const u32* ids; u32 n; };
ST_DEV LgList lgrid_list(const LightGridDev& lg, float3 p) {
    LgList all; all.ids = nullptr; all.n = lg.light_count;
    if (!(isfinite(p.x) && isfinite(p.y) && isfinite(p.z))) return all;
    const u32 ncell = lg.dims[0] * lg.dims[1] * lg.dims[2];
    u32 cell = ncell;   // the outside list
    if (ncell > 0u) {
        const float pc[3] = {p.x, p.y, p.z};
        u32 idx[3]; bool inside = true;
#pragma unroll
        for (int a = 0; a < 3; a++) {
            const float t = xmul(xsub(pc[a], lg.lo[a]), lg.inv_cell[a]);
            if (!(t >= -lg.band[a]) || !(t < xadd((float)lg.dims[a], lg.band[a]))) inside = false;
            const int i = (int)floorf(fminf(fmaxf(t, 0.0f), (float)(lg.dims[a] - 1u)));
            idx[a] = (u32)i;
        }
        if (inside) cell = (idx[2] * lg.dims[1] + idx[1]) * lg.dims[0] + idx[0];
    }
    const u32 c = __ldg(lg.counts + cell);
    if (c == kLightGridOverflow) return all;
    LgList l; l.ids = lg.lists + (size_t)cell * kLightGridK; l.n = c;
    return l;
}
ST_DEV u32 lgrid_pick(const LgList& l, u32 r) { return l.ids ? __ldg(l.ids + r) : r; }
// ephemeral_build over a list of n slots: min(n, 16) uniform draws from the list at ipdf = n (the option off: the list of every slot)
ST_DEV EphRes ephemeral_build_list(Rng& rng, const SceneDev& sc, const Hit& hit, const LgList& list) {
    EphRes res; res.m = 0.f; res.w = 0.f; res.light_id = 0u; res.rad = lightrad_zero();
    float res_pdf = 0.0f;
    u32 lc = list.n;
    u32 max_samples = lc < 16u ? lc : 16u;
    float ipdf = (float)lc;
    for (u32 nth = 0u; nth < max_samples; nth++) {
        u32 id = lgrid_pick(list, rng_u32(rng) % lc);
        LightRad lr = light_radiance(light_load(sc, id), hit);
        float pdf = sqrtf(luma(lr.radiance));
        float weight = pdf * ipdf;
        res.m += 1.0f; res.w += weight;
        if (rng_f(rng) * res.w < weight) { res.light_id = id; res.rad = lr; res_pdf = pdf; }
    }
    res.w = res_norm(res.w, res_pdf, 1.0f, res.m);
    return res;
}

// Mis (mis.rs:12-155)
struct MisIn { float lhs_m, rhs_m, rhs_jacobian, lhs_lhs_pdf, lhs_rhs_pdf, rhs_lhs_pdf, rhs_rhs_pdf; };
struct MisOut { float m, lhs_pdf, lhs_mis, rhs_pdf, rhs_mis; };
ST_DEV float mis_ratio(float x, float y) { float s = x + y; return (s == 0.0f) ? 0.0f : x / s; }
ST_DEV float mis_conf(float q0, float q1) { return (q0 <= 0.0f) ? 1.0f : sat(pow_det(rmin(q1 / q0, 1.0f), 8.0f)); }
ST_DEV MisOut mis_eval(const MisIn& s) {
    MisOut r;
    r.m = s.rhs_m * rmin(mis_conf(s.rhs_rhs_pdf, s.rhs_lhs_pdf), mis_conf(s.lhs_rhs_pdf, s.lhs_lhs_pdf));
    float t = mis_ratio(s.lhs_m, s.rhs_m);
    r.lhs_mis = t + (1.0f - t) * mis_ratio(s.lhs_m * s.lhs_lhs_pdf, s.rhs_m * s.lhs_rhs_pdf);
    r.rhs_mis = (1.0f - t) * mis_ratio(s.rhs_m * s.rhs_rhs_pdf * s.rhs_jacobian, s.lhs_m * s.rhs_lhs_pdf);
    r.lhs_pdf = s.lhs_lhs_pdf; r.rhs_pdf = s.rhs_lhs_pdf;
    return r;
}

// checkerboard helpers (utils.rs:33-43), GI cadence (frame.rs:19-21)
ST_DEV uint2 checker(u32 gx, u32 gy, u32 frame) { return make_uint2(gx * 2u + ((frame + gy) % 2u), gy); }
ST_DEV bool checker_at(u32 px, u32 py, u32 frame) { uint2 r = checker(px / 2u, py, frame); return r.x == px && r.y == py; }
ST_DEV bool gi_tracing_frame(u32 frame) { return frame % 6u < 4u; }

}  // namespace ST_NS
