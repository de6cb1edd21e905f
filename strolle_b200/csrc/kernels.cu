// strolle_b200 — sm_90a (H100) kernels for the per-pixel GI hot path.
//
// One kernel per reference compute entry point (strolle-shaders/src/*.rs, K1–K22 in
// SURVEY.md §2.2) plus the primary-visibility G-buffer kernel that replaces the rasteriser
// and the composition kernel.  All kernels are HBM/latency-bound integer+f32 work: no tensor
// cores.  Mapping: one thread per pixel, CTAs of 128 threads covering a 16x8 pixel tile so
// that a warp reads two 256-byte row segments of every float4 texture (coalesced 16-byte
// loads); BVH nodes / triangles go through the read-only path (ld.global.nc.v4.f32) and the
// traversal stack lives in shared memory, one conflict-free column per thread.
#include <algorithm>
#include <cstdio>
#include <cuda_fp16.h>
#include <cuda.h>   // CUtensorMap (type only; the encoder is reached through cudaGetDriverEntryPoint)
#include <map>
#include <mutex>
#include <tuple>
#include <vector>
#include "st_device.cuh"
#include "kernels.h"
#if ST_BLOOM_TAIL_KIND == 2
#include <cooperative_groups.h>
#endif

// Compiled twice (strolle_b200/build.py): as namespace st with strict IEEE arithmetic (every kernel), and with -DST_FAST=1 as
// namespace stf, the fast-shading flavour of the ReSTIR kernels K5-K19 only (see st_math.cuh).
#if defined(ST_FAST) && ST_FAST
#define ST_EXACT_ONLY 0
#else
#define ST_EXACT_ONLY 1
#endif

namespace ST_NS {

#define TILE_W 16
#define TILE_H 8

struct Px { u32 x, y; bool in; };
// Row tile of this CTA.  In a strip that mirrors rows into the strip below it, the CTAs are rotated so that the bottom boundary rows are
// computed FIRST (the top boundary rows follow, the interior last): the remote stores of both boundaries drain over NVLink while the
// interior is still computing, instead of at the very end of the kernel.
ST_DEV u32 row_tile(const CameraDev& cam) {
    if (cam.mirror_dn == 0) return blockIdx.y;
    const u32 lead = (u32)(ST_REACH_SPATIAL / TILE_H);
    return gridDim.y > lead ? (blockIdx.y + gridDim.y - lead) % gridDim.y : blockIdx.y;
}
ST_DEV Px pixel_full(const CameraDev& cam) {
    Px p; p.x = blockIdx.x * TILE_W + (threadIdx.x % TILE_W); p.y = (u32)cam.y0 + row_tile(cam) * TILE_H + (threadIdx.x / TILE_W);
    p.in = p.x < (u32)cam.w && p.y < (u32)cam.y1;
    return p;
}
// half-width checkerboard dispatch of the reference: gid.x < 8*(((W+7)/8)/2), gid.y < 8*((H+7)/8)
ST_DEV int half_grid_w(int w) { return 8 * (((w + 7) / 8) / 2); }
ST_DEV Px pixel_half(const CameraDev& cam) {
    Px p; p.x = blockIdx.x * TILE_W + (threadIdx.x % TILE_W); p.y = (u32)cam.y0 + row_tile(cam) * TILE_H + (threadIdx.x / TILE_W);
    p.in = p.x < (u32)half_grid_w(cam.w) && p.y < (u32)cam.y1;
    return p;
}
ST_DEV size_t pix(const CameraDev& cam, u32 x, u32 y) { return (size_t)y * (size_t)cam.w + x; }
ST_DEV size_t screen_idx(const CameraDev& cam, u32 x, u32 y) { return (size_t)(y * to_u32_sat(cam.curr.screen.x) + x); }   // camera.rs:39-41 (u32 arithmetic)
ST_DEV bool in_tex(const CameraDev& cam, u32 x, u32 y) { return x < (u32)cam.w && y < (u32)cam.h; }
ST_DEV float4 tex_or_zero(const float4* __restrict__ t, const CameraDev& cam, u32 x, u32 y) { return in_tex(cam, x, y) ? t[pix(cam, x, y)] : f4zero(); }
ST_DEV void tex_store(float4* __restrict__ t, const CameraDev& cam, u32 x, u32 y, float4 v) { if (in_tex(cam, x, y)) t[pix(cam, x, y)] = v; }
ST_DEV Hit load_hit(const GpuCamera& c, const float4* __restrict__ d0, const float4* __restrict__ d1, const CameraDev& cam, u32 x, u32 y) {
    return hit_make(cam_ray(c, x, y), gbuf_unpack(tex_or_zero(d0, cam, x, y), tex_or_zero(d1, cam, x, y)));
}
// variant whose base colour comes from the byte table (kernels that consume hit.g.base_color)
ST_DEV Hit load_hit_lut(const SceneDev& sc, const GpuCamera& c, const float4* __restrict__ d0, const float4* __restrict__ d1, const CameraDev& cam, u32 x, u32 y) {
    return hit_make(cam_ray(c, x, y), gbuf_unpack(sc, tex_or_zero(d0, cam, x, y), tex_or_zero(d1, cam, x, y)));
}
#define ST_TRACE_STACK()                                          \
    __shared__ u32 s_stack[ST_BVH_STACK * ST_BLOCK];              \
    TraceStack stk; stk.base = s_stack + threadIdx.x;

#define KPARAMS const __grid_constant__ CameraDev cam, const __grid_constant__ SceneDev sc

// Launch bounds per kernel: ST_LB_<KERNEL> is __launch_bounds__(128) (ptxas' own register choice) unless a minimum number
// of resident CTAs per SM is set (ST_MINB_<KERNEL> = N caps registers at 65536 / (128 N)); values checked on an H100 with
// tools/occupancy_tune.py.  -DST_MINB_ALL=N overrides every kernel at once (tuning builds).
#define ST_LB_N(N) __launch_bounds__(ST_BLOCK, N)
// these five run at 8 CTAs/SM (64 registers; di_temporal at 12, 40 registers); on an H100 the frame is within 1 % of uncapped and of
// capping every kernel at 8 CTAs/SM, while capping every kernel at 12 is 26 % slower (Cornell 1080p, DESIGN.md §4)
#if !defined(ST_MINB_ALL)
#define ST_MINB_GI_PREVIEW 8
#define ST_MINB_GI_TEMPORAL 8
#define ST_MINB_GI_SAMPLING_B 8
#define ST_MINB_GI_SPATIAL_PICK 8
#define ST_MINB_DI_TEMPORAL 12
#endif
// ST_LB_<K>: -DST_MINB_ALL=N beats a per-kernel ST_MINB_<K>, which beats ptxas' own choice.  The preprocessor cannot test a macro whose
// name is pasted together, so the three-way choice is spelled once per kernel through ST_LB_PICK (0 = "no minimum").
#define ST_LB_PICK(per_kernel) ST_LB_CHOOSE(ST_MINB_ALL_OR_0, per_kernel)
#if defined(ST_MINB_ALL)
#define ST_MINB_ALL_OR_0 ST_MINB_ALL
#else
#define ST_MINB_ALL_OR_0 0
#endif
template <int ALL, int ONE> struct LbMin { static constexpr int value = ALL > 0 ? ALL : ONE; };
#define ST_LB_CHOOSE(all, one) __launch_bounds__(ST_BLOCK, (LbMin<all, one>::value > 0 ? LbMin<all, one>::value : 1))
#ifndef ST_MINB_PRIM_GBUFFER
#define ST_MINB_PRIM_GBUFFER 0
#endif
#define ST_LB_PRIM_GBUFFER ST_LB_PICK(ST_MINB_PRIM_GBUFFER)
#ifndef ST_MINB_DI_SAMPLING
#define ST_MINB_DI_SAMPLING 0
#endif
#define ST_LB_DI_SAMPLING ST_LB_PICK(ST_MINB_DI_SAMPLING)
#ifndef ST_MINB_DI_TEMPORAL
#define ST_MINB_DI_TEMPORAL 0
#endif
#define ST_LB_DI_TEMPORAL ST_LB_PICK(ST_MINB_DI_TEMPORAL)
#ifndef ST_MINB_DI_SPATIAL_PICK
#define ST_MINB_DI_SPATIAL_PICK 0
#endif
#define ST_LB_DI_SPATIAL_PICK ST_LB_PICK(ST_MINB_DI_SPATIAL_PICK)
#ifndef ST_MINB_SPATIAL_TRACE
#define ST_MINB_SPATIAL_TRACE 0
#endif
#define ST_LB_SPATIAL_TRACE ST_LB_PICK(ST_MINB_SPATIAL_TRACE)
#ifndef ST_MINB_DI_RESOLVING
#define ST_MINB_DI_RESOLVING 0
#endif
#define ST_LB_DI_RESOLVING ST_LB_PICK(ST_MINB_DI_RESOLVING)
#ifndef ST_MINB_GI_SAMPLING_A
#define ST_MINB_GI_SAMPLING_A 0
#endif
#define ST_LB_GI_SAMPLING_A ST_LB_PICK(ST_MINB_GI_SAMPLING_A)
#ifndef ST_MINB_GI_SAMPLING_B
#define ST_MINB_GI_SAMPLING_B 0
#endif
#define ST_LB_GI_SAMPLING_B ST_LB_PICK(ST_MINB_GI_SAMPLING_B)
#ifndef ST_MINB_GI_TEMPORAL
#define ST_MINB_GI_TEMPORAL 0
#endif
#define ST_LB_GI_TEMPORAL ST_LB_PICK(ST_MINB_GI_TEMPORAL)
#ifndef ST_MINB_GI_SPATIAL_PICK
#define ST_MINB_GI_SPATIAL_PICK 0
#endif
#define ST_LB_GI_SPATIAL_PICK ST_LB_PICK(ST_MINB_GI_SPATIAL_PICK)
#ifndef ST_MINB_GI_SPATIAL_SAMPLE
#define ST_MINB_GI_SPATIAL_SAMPLE 0
#endif
#define ST_LB_GI_SPATIAL_SAMPLE ST_LB_PICK(ST_MINB_GI_SPATIAL_SAMPLE)
#ifndef ST_MINB_GI_PREVIEW
#define ST_MINB_GI_PREVIEW 0
#endif
#define ST_LB_GI_PREVIEW ST_LB_PICK(ST_MINB_GI_PREVIEW)
#ifndef ST_MINB_GI_RESOLVING
#define ST_MINB_GI_RESOLVING 0
#endif
#define ST_LB_GI_RESOLVING ST_LB_PICK(ST_MINB_GI_RESOLVING)

#if ST_EXACT_ONLY
// ---------------------------------------------------------------------------------------------
// Primary-visibility G-buffer (stands in for strolle-shaders/src/prim_raster.rs:41-128; SURVEY §8f-1)
// ---------------------------------------------------------------------------------------------
ST_DEV float4 frame_reprojection_px(const CameraDev& cam, int cur, Px p, float4 surface_texel, float4 vel);
// `with_reprojection` (ST_OPT_FUSED_PASSES; single GPU, or a strip on a frame where nothing moved): K4 runs in this launch too — its inputs for the pixel are still in registers
// NMAP (ST_OPT_NORMAL_MAPS, only while some material has a normal map): the shading normal is the mapped one (nmap_normal)
// TEXF (ST_OPT_TEXTURE_FILTER, only while some material has a colour texture): the material's textures are filtered (texf_sample)
template <bool NMAP, bool TEXF>
__global__ void ST_LB_PRIM_GBUFFER k_prim_gbuffer(KPARAMS, int cur, int with_reprojection, const __grid_constant__ TexFilterDev tf) {
    ST_TRACE_STACK();
    Px p = pixel_full(cam);
    if (!p.in) return;
    Ray ray = cam_ray(cam.curr, p.x, p.y);
    TriHit th = trace_closest(ray, sc, stk);
    if ((int)p.y < cam.own_y0 || (int)p.y >= cam.own_y1) uncount_ray(sc);   // a neighbour's row, recomputed here: not counted as a ray of the frame
    float4 g0 = f4zero(), g1 = f4zero(), surf = f4zero(), vel = f4zero(), tid = f4(bitsf(0xffffffffu), 0.f, 0.f, 0.f), nd = f4zero();
    if (trihit_some(th)) {
        const GpuMaterial m = sc.materials[th.material_id];
        if (NMAP) th.normal = nmap_normal(sc, th, m.normal_map_texture);
        GBuf g;
        float2 mr;
        if (TEXF) {
            TexFoot ft; ft.tri = th.triangle_id; ft.dir = ray.d; ft.w = texf_cone_width(cam.curr, p.x, p.y, th.t, true);
            const float4 t = texf_sample(sc, tf, th.material_id, 2u, m.metallic_roughness_texture, f4(1.0f, m.roughness, m.metallic, 1.0f), th.uv, ft);
            mr = f2(t.z, t.y);
            g.base_color = texf_sample(sc, tf, th.material_id, 0u, m.base_color_texture, m.base_color, th.uv, ft);
            g.emissive = xyz(texf_sample(sc, tf, th.material_id, 1u, m.emissive_texture, m.emissive, th.uv, ft));
        } else {
            mr = mat_metallic_roughness(sc, m, th.uv);
            g.base_color = mat_base_color(sc, m, th.uv); g.emissive = mat_emissive(sc, m, th.uv);
        }
        g.normal = th.normal; g.metallic = mr.x;
        g.roughness = mr.y; g.reflectance = m.reflectance; g.depth = dist(ray.o, th.point);
        // untextured base colour: its gamma-encoded bytes come from the per-material table
        gbuf_pack_pre(g, all_zero(m.base_color_texture) ? __ldg(sc.material_packed + th.material_id) : gbuf_pack_color(g.base_color), &g0, &g1);
        float2 n = oct_encode(th.normal);
        surf = f4(n.x, n.y, g.depth, m.roughness);
        nd = f4(oct_decode(n), g.depth);   // what every consumer of the surface map decodes, computed once
        // prim_raster::vs (prim_raster.rs:25-34): where this surface point was last frame, per instance
        const float4* xf = sc.instance_xforms + 6u * (size_t)__ldg(sc.tri_instance + th.triangle_id);
        float4 c0 = ldg4(xf), c1 = ldg4(xf + 1), c2 = ldg4(xf + 2), q0 = ldg4(xf + 3), q1 = ldg4(xf + 4), q2 = ldg4(xf + 5);
        float3 local = ((xyz(c0) * th.point.x + xyz(c1) * th.point.y) + xyz(c2) * th.point.z) + f3(c0.w, c1.w, c2.w);
        float3 prev_point = ((xyz(q0) * local.x + xyz(q1) * local.y) + xyz(q2) * local.z) + f3(q0.w, q1.w, q2.w);
        float2 v = cam_world_to_screen(cam.curr, th.point) - cam_world_to_screen(cam.prev, prev_point);
        if (len2(v) >= 0.001f) vel = f4(v.x, v.y, 0.f, 0.f);
        tid.x = bitsf(th.triangle_id);
        // strip partition: which rows of LAST frame's buffers the temporal passes (K4, K6, K11, K14, K20) of this strip will read:
        // they fetch at prev = pixel - velocity (rounded, or its floor/ceil corners).  Only pixels whose reprojection leaves the
        // owned rows report; the pull kernel that follows brings exactly those rows in from their owners.
        if (cam.need_rows != nullptr && vel.y != 0.0f && (int)p.y >= cam.own_y0 && (int)p.y < cam.own_y1) {
            float py = (float)p.y - vel.y;
            int lo = max(0, min(cam.h - 1, to_i32_sat(floorf(py)))), hi = max(0, min(cam.h - 1, to_i32_sat(ceilf(py))));
            if (lo < cam.own_y0) atomicMin(cam.need_rows, lo);
            if (hi >= cam.own_y1) atomicMax(cam.need_rows + 1, hi);
        }
    }
    size_t i = pix(cam, p.x, p.y);
    cam.prim_gbuffer_d0[cur][i] = g0; cam.prim_gbuffer_d1[cur][i] = g1; cam.prim_surface_map[cur][i] = surf;
    cam.velocity_map[i] = vel; cam.prim_triangle_ids[i] = tid; cam.surface_nd[i] = nd;
    if (with_reprojection && (int)p.y >= cam.own_y0 && (int)p.y < cam.own_y1) cam.reprojection_map[i] = frame_reprojection_px(cam, cur, p, surf, vel);   // not for the rows a strip recomputes beyond its own
}

// K4 frame_reprojection::main (frame_reprojection.rs:7-95): where the pixel was last frame and how far that can be trusted
ST_DEV float4 frame_reprojection_px(const CameraDev& cam, int cur, Px p, float4 surface_texel, float4 vel) {
    const float4* sp_ = cam.prim_surface_map[cur ^ 1];
    Reproj rp; rp.px = 0.f; rp.py = 0.f; rp.confidence = 0.f; rp.validity = 0u;
    Surf surface = surf_decode(surface_texel);
    if (surface.depth == 0.0f) return reproj_encode(rp);
    float2 prev = f2((float)p.x, (float)p.y) - f2(vel.x, vel.y);
    float2 pr = f2(roundf(prev.x), roundf(prev.y));
    if (cam_contains_f(cam.prev, pr)) {
        Surf ps = surf_decode(tex_or_zero(sp_, cam, to_u32_sat(pr.x), to_u32_sat(pr.y)));
        float conf = surf_similarity(ps, surface);
        if (conf > 0.0f) { rp.px = prev.x; rp.py = prev.y; rp.confidence = conf; rp.validity = 0u; }
    }
    if (reproj_some(rp)) {
        int x0 = to_i32_sat(floorf(rp.px)), x1 = to_i32_sat(ceilf(rp.px)), y0 = to_i32_sat(floorf(rp.py)), y1 = to_i32_sat(ceilf(rp.py));
        int xs[4] = {x0, x1, x0, x1}, ys[4] = {y0, y0, y1, y1};
#pragma unroll
        for (int k = 0; k < 4; k++) {
            if (!cam_contains_i(cam.curr, xs[k], ys[k])) continue;
            if (surf_similarity(surf_decode(sp_[pix(cam, (u32)xs[k], (u32)ys[k])]), surface) >= 0.25f) rp.validity |= (1u << k);
        }
    }
    return reproj_encode(rp);
}
__global__ void __launch_bounds__(ST_BLOCK) k_frame_reprojection(KPARAMS, int cur) {
    Px p = pixel_full(cam);
    if (!p.in) return;
    size_t i = pix(cam, p.x, p.y);
    cam.reprojection_map[i] = frame_reprojection_px(cam, cur, p, cam.prim_surface_map[cur][i], cam.velocity_map[i]);
}
#endif   // ST_EXACT_ONLY

// K5 di_sampling::main (di_sampling.rs:4-94): the initial sample of a pixel whose primary hit is `hit`
// LGRID (ST_OPT_LIGHT_GRID): the candidates are drawn from the light grid's list for hit.point instead of from every slot
template <bool LGRID>
ST_DEV DiRes di_sampling_px(const CameraDev& cam, const SceneDev& sc, const TraceStack& stk, const Hit& hit, u32 seed, u32 frame, Px p, const LightGridDev& lg) {
    Rng rng = rng_make(seed, p.x, p.y);
    EphRes res = LGRID ? ephemeral_build_list(rng, sc, hit, lgrid_list(lg, hit.point)) : ephemeral_build(rng, sc, hit);
    DiRes out = di_zero();
    if (res.m > 0.0f) {
        float4 bn = blue_noise(sc, p.x, p.y, frame);
        Ray ray = light_ray_bnoise(light_load(sc, res.light_id), f2(bn.x, bn.y), hit.point);
        bool occ = trace_any(ray, sc, stk);
        if (occ) res.w = 0.0f;
        out.pdf = 0.f; out.confidence = 0.f; out.light_id = res.light_id; out.light_point = ray.o; out.occluded = occ; out.m = 1.0f; out.w = res.w;
    }
    return out;
}
template <bool LGRID>
__global__ void ST_LB_DI_SAMPLING k_di_sampling(KPARAMS, int cur, u32 seed, u32 frame, const __grid_constant__ LightGridDev lg) {
    ST_TRACE_STACK();
    Px p = pixel_full(cam);
    if (!p.in) return;
    Hit hit = load_hit_lut(sc, cam.curr, cam.prim_gbuffer_d0[cur], cam.prim_gbuffer_d1[cur], cam, p.x, p.y);
    if (!hit_some(hit)) return;
    di_store(di_sampling_px<LGRID>(cam, sc, stk, hit, seed, frame, p, lg), cam.di_reservoirs[1], screen_idx(cam, p.x, p.y));
}

// K6 di_temporal_resampling::main (di_temporal_resampling.rs:4-112): merges this frame's sample `lhs` with last frame's reservoir at
// the reprojected position
ST_DEV DiRes di_temporal_px(const CameraDev& cam, const SceneDev& sc, int cur, u32 seed, Px p, const Hit& lhs_hit, DiRes lhs) {
    size_t npx = (size_t)cam.w * cam.h;
    Rng rng = rng_make(seed, p.x, p.y);
    if (lhs.m != 0.0f) lhs.pdf = di_pdf_with(lhs, light_load(sc, lhs.light_id), lhs_hit);
    DiRes rhs = di_zero();
    Hit rhs_hit = hit_zero();
    bool killed = false;
    Reproj rp = reproj_decode(cam.reprojection_map[pix(cam, p.x, p.y)]);
    if (reproj_some(rp)) {
        uint2 rpos = reproj_round(rp);
        size_t ridx = screen_idx(cam, rpos.x, rpos.y);
        if (ridx < npx) rhs = di_load(cam.di_reservoirs[0], ridx);
        rhs.m = rmin(rhs.m, 64.0f);
        if (rhs.m != 0.0f) {
            GpuLight rl = light_load(sc, rhs.light_id);
            u32 slot = fbits(rl.d3.x);
            if (slot == 0xcafebabeu) { rhs.w = 0.0f; killed = true; }
            else if (slot > 0u) rhs.light_id = slot - 1u;
            rhs_hit = load_hit_lut(sc, cam.prev, cam.prim_gbuffer_d0[cur ^ 1], cam.prim_gbuffer_d1[cur ^ 1], cam, rpos.x, rpos.y);
        }
    }
    MisIn mi;
    mi.lhs_m = lhs.m; mi.rhs_m = rhs.m; mi.rhs_jacobian = 1.0f; mi.lhs_lhs_pdf = lhs.pdf; mi.rhs_rhs_pdf = rhs.pdf;
    mi.lhs_rhs_pdf = ((lhs.m > 0.0f) & hit_some(rhs_hit)) ? di_pdf_with(lhs, light_prev(light_load(sc, lhs.light_id)), rhs_hit) : 0.0f;
    mi.rhs_lhs_pdf = ((rhs.m > 0.0f) & !killed) ? di_pdf_with(rhs, light_load(sc, rhs.light_id), lhs_hit) : 0.0f;
    MisOut mo = mis_eval(mi);
    DiRes main_ = di_zero();
    float main_pdf = 0.0f;
    if (di_update(main_, rng, lhs, mo.lhs_mis * mo.lhs_pdf * lhs.w)) main_pdf = mo.lhs_pdf;
    if (di_update(main_, rng, rhs, mo.rhs_mis * mo.rhs_pdf * rhs.w)) main_pdf = mo.rhs_pdf;
    main_.m = lhs.m + mo.m;
    main_.pdf = main_pdf;
    main_.confidence = killed ? 0.0f : 1.0f;
    main_.w = res_norm(main_.w, main_pdf, 1.0f, 1.0f);
    return main_;
}
__global__ void ST_LB_DI_TEMPORAL k_di_temporal(KPARAMS, int cur, u32 seed) {
    Px p = pixel_full(cam);
    if (!p.in) return;
    size_t lhs_idx = screen_idx(cam, p.x, p.y);
    Hit lhs_hit = load_hit_lut(sc, cam.curr, cam.prim_gbuffer_d0[cur], cam.prim_gbuffer_d1[cur], cam, p.x, p.y);
    if (!hit_some(lhs_hit)) return;
    di_store_m(cam, di_temporal_px(cam, sc, cur, seed, p, lhs_hit, di_load(cam.di_reservoirs[1], lhs_idx)), cam.di_reservoirs[1], lhs_idx, p.y, cam.di_mirror_reach);
}
// K5 + K6 in one launch (ST_OPT_FUSED_PASSES): the pixel's fresh sample goes from K5 to K6 in registers instead of through di_reservoirs[1]
// (the hit is decoded once).  What di_store / di_load would do to the sample on the way (confidence -> byte) is the identity for K5's
// output (confidence 0), so the result is the two-launch result bit for bit.
template <bool LGRID>
__global__ void ST_LB_DI_SAMPLING k_di_sample_temporal(KPARAMS, int cur, u32 seed_sampling, u32 seed_temporal, u32 frame, const __grid_constant__ LightGridDev lg) {
    ST_TRACE_STACK();
    Px p = pixel_full(cam);
    if (!p.in) return;
    Hit hit = load_hit_lut(sc, cam.curr, cam.prim_gbuffer_d0[cur], cam.prim_gbuffer_d1[cur], cam, p.x, p.y);
    if (!hit_some(hit)) return;
    DiRes fresh = di_sampling_px<LGRID>(cam, sc, stk, hit, seed_sampling, frame, p, lg);
    di_store_m(cam, di_temporal_px(cam, sc, cur, seed_temporal, p, hit, fresh), cam.di_reservoirs[1], screen_idx(cam, p.x, p.y), p.y, cam.di_mirror_reach);
}

// The four scratch texels of one checkerboard pair: (d0, d1) of texel a = (2gx, gy) and texel b = (2gx + 1, gy).
// state 0: the pair has no left-hand pixel on the screen, nothing is written; 1: only the two d1 texels are cleared; 2: all four.
struct PairTexels { float4 a0, a1, b0, b1; int state; };

// K7 di_spatial_resampling::pick (di_spatial_resampling.rs:4-147); scratch buf_d0 = di_diff_samples,
// buf_d1 = di_diff_curr_colors (passes/di_spatial_resampling.rs:24-28).  Sky pixels clear buf_d1
// (the reference leaves stale texels there and later reads out of bounds — SURVEY Appendix C-15).
ST_DEV PairTexels di_spatial_pick_pair(const CameraDev& cam, const SceneDev& sc, int cur, u32 seed, u32 frame, Px g) {
    PairTexels o; o.a0 = o.a1 = o.b0 = o.b1 = f4zero(); o.state = 0;
    uint2 lp = checker(g.x, g.y, frame / 2u + 1u);
    if (!cam_contains_u(cam.curr, lp.x, lp.y)) return o;
    o.state = 1;
    size_t lhs_idx = screen_idx(cam, lp.x, lp.y);
    Rng rng = rng_make(seed, lp.x, lp.y);
    const float4* gd0 = cam.prim_gbuffer_d0[cur]; const float4* gd1 = cam.prim_gbuffer_d1[cur];
    Hit lhs_hit = load_hit_lut(sc, cam.curr, gd0, gd1, cam, lp.x, lp.y);
    if (!hit_some(lhs_hit)) return o;
    DiRes lhs = di_load(cam.di_reservoirs[1], lhs_idx);
    DiRes rhs = di_zero();
    size_t rhs_idx = 0;
    Hit rhs_hit = hit_zero();
    float max_radius = 128.0f;
    for (u32 nth = 0u; nth < 8u; nth++) {
        float2 off = rng_disk(rng) * max_radius;
        float2 fp = f2((float)lp.x, (float)lp.y) + off;
        uint2 rpos = cam_contain(cam.curr, to_i32_sat(fp.x), to_i32_sat(fp.y));
        if (rpos.x == lp.x && rpos.y == lp.y) continue;
        // the rejection tests only need the neighbour's depth and normal: one (normal, depth) float4
        float4 nd = tex_or_zero(cam.surface_nd, cam, rpos.x, rpos.y);
        if (nd.w == 0.0f) { max_radius = rmax(max_radius * 0.5f, 5.0f); continue; }
        if (fabs_(nd.w - lhs_hit.g.depth) > 0.33f * lhs_hit.g.depth) { max_radius = rmax(max_radius * 0.5f, 5.0f); continue; }
        if (dot(xyz(nd), lhs_hit.g.normal) < 0.33f) { max_radius = rmax(max_radius * 0.5f, 5.0f); continue; }
        rhs_idx = screen_idx(cam, rpos.x, rpos.y);
        rhs = di_load(cam.di_reservoirs[1], rhs_idx);
        if (rhs.m != 0.0f) { rhs_hit = load_hit_lut(sc, cam.curr, gd0, gd1, cam, rpos.x, rpos.y); break; }
    }
    if (rhs.m == 0.0f) return o;
    float lhs_rhs_pdf = di_pdf_with(lhs, light_load(sc, lhs.light_id), rhs_hit);
    float rhs_lhs_pdf = di_pdf_with(rhs, light_load(sc, rhs.light_id), lhs_hit);
    Ray ra = (lhs_rhs_pdf > 0.0f) ? di_ray(lhs, rhs_hit.point) : ray_zero();
    Ray rb = (rhs_lhs_pdf > 0.0f) ? di_ray(rhs, lhs_hit.point) : ray_zero();
    float2 na = oct_encode(ra.d), nb = oct_encode(rb.d);
    o.a0 = f4(ra.o, ra.len); o.a1 = f4(na.x, na.y, bitsf((u32)rhs_idx + 1u), 0.0f);
    o.b0 = f4(rb.o, rb.len); o.b1 = f4(nb.x, nb.y, lhs_rhs_pdf, rhs_lhs_pdf);
    o.state = 2;
    return o;
}
ST_DEV void store_pair_texels(const CameraDev& cam, const PairTexels& o, float4* buf_d0, float4* buf_d1, Px g) {
    if (o.state == 0) return;
    u32 ax = g.x * 2u, bx = g.x * 2u + 1u;
    if (o.state == 2) { tex_store(buf_d0, cam, ax, g.y, o.a0); tex_store(buf_d0, cam, bx, g.y, o.b0); }
    tex_store(buf_d1, cam, ax, g.y, o.a1); tex_store(buf_d1, cam, bx, g.y, o.b1);
}
__global__ void ST_LB_DI_SPATIAL_PICK k_di_spatial_pick(KPARAMS, int cur, u32 seed, u32 frame) {
    Px g = pixel_half(cam);
    if (!g.in) return;
    store_pair_texels(cam, di_spatial_pick_pair(cam, sc, cur, seed, frame, g), cam.di_diff_samples, cam.di_diff_curr_colors, g);
}

// K8 / K16 *_spatial_resampling::trace (di_spatial_resampling.rs:150-209, gi_spatial_resampling.rs:163-222): one scratch texel
ST_DEV float4 spatial_trace_texel(const SceneDev& sc, const TraceStack& stk, float4 d0, float4 d1) {
    if (all_zero(d1)) return f4zero();
    Ray ray = ray_make(xyz(d0), oct_decode(f2(d1.x, d1.y)), d0.w);
    bool occ = trace_any(ray, sc, stk);
    return f4(occ ? 0.0f : 1.0f, d1.z, d1.w, 0.0f);
}
__global__ void ST_LB_SPATIAL_TRACE k_spatial_trace(KPARAMS, const float4* __restrict__ buf_d0, const float4* __restrict__ buf_d1, float4* __restrict__ buf_d2) {
    ST_TRACE_STACK();
    Px p = pixel_full(cam);
    if (!p.in) return;
    size_t i = pix(cam, p.x, p.y);
    buf_d2[i] = spatial_trace_texel(sc, stk, buf_d0[i], buf_d1[i]);
}
// the two visibility texels of a pair as K8 / K16 would leave them for K9 / K17 (a texel outside the texture reads as zero)
ST_DEV void trace_pair_texels(const CameraDev& cam, const SceneDev& sc, const TraceStack& stk, const PairTexels& o, Px g, float4* d2a, float4* d2b) {
    u32 ax = g.x * 2u, bx = g.x * 2u + 1u;
    *d2a = (o.state == 2 && in_tex(cam, ax, g.y)) ? spatial_trace_texel(sc, stk, o.a0, o.a1) : f4zero();
    *d2b = (o.state == 2 && in_tex(cam, bx, g.y)) ? spatial_trace_texel(sc, stk, o.b0, o.b1) : f4zero();
}

// K9 di_spatial_resampling::sample (di_spatial_resampling.rs:212-297); d0 / d1 = the pair's two visibility texels
ST_DEV void di_spatial_sample_pair(const CameraDev& cam, u32 seed, u32 frame, Px g, float4 d0, float4 d1) {
    uint2 lp = checker(g.x, g.y, frame / 2u + 1u);
    if (!cam_contains_u(cam.curr, lp.x, lp.y)) return;
    size_t npx = (size_t)cam.w * cam.h;
    size_t lhs_idx = screen_idx(cam, lp.x, lp.y);
    Rng rng = rng_make(seed, lp.x, lp.y);
    const float4* in = cam.di_reservoirs[1]; float4* out = cam.di_reservoirs[2];
    float lhs_rhs_vis = d0.x; u32 rhs_idx = fbits(d0.y);
    float rhs_lhs_vis = d1.x, lhs_rhs_pdf = d1.y, rhs_lhs_pdf = d1.z;
    DiRes lhs = di_load(in, lhs_idx);
    if (rhs_idx > 0u && (size_t)rhs_idx - 1 < npx) {
        DiRes rhs = di_load(in, (size_t)rhs_idx - 1);
        MisIn mi;
        mi.lhs_m = lhs.m; mi.rhs_m = rhs.m; mi.rhs_jacobian = 1.0f; mi.lhs_lhs_pdf = lhs.pdf;
        mi.lhs_rhs_pdf = lhs_rhs_pdf * lhs_rhs_vis; mi.rhs_lhs_pdf = rhs_lhs_pdf * rhs_lhs_vis; mi.rhs_rhs_pdf = rhs.pdf;
        MisOut mo = mis_eval(mi);
        DiRes main_ = di_zero();
        float main_pdf = 0.0f;
        if (di_update(main_, rng, lhs, mo.lhs_mis * mo.lhs_pdf * lhs.w)) main_pdf = mo.lhs_pdf;
        if (di_update(main_, rng, rhs, mo.rhs_mis * mo.rhs_pdf * rhs.w)) { main_pdf = mo.rhs_pdf; main_.occluded = lhs_rhs_vis == 0.0f; }
        main_.m = lhs.m + mo.m;
        main_.pdf = main_pdf;
        main_.w = res_norm(main_.w, main_pdf, 1.0f, 1.0f);
        di_store(main_, out, lhs_idx);
    } else di_store(lhs, out, lhs_idx);
    uint2 op = checker(g.x, g.y, frame / 2u);
    if (cam_contains_u(cam.curr, op.x, op.y)) { size_t oi = screen_idx(cam, op.x, op.y); di_store(di_load(in, oi), out, oi); }
}
__global__ void __launch_bounds__(ST_BLOCK) k_di_spatial_sample(KPARAMS, u32 seed, u32 frame) {
    Px g = pixel_half(cam);
    if (!g.in) return;
    di_spatial_sample_pair(cam, seed, frame, g, tex_or_zero(cam.di_diff_stash, cam, g.x * 2u, g.y), tex_or_zero(cam.di_diff_stash, cam, g.x * 2u + 1u, g.y));
}
// K7 + K8 + K9 in one launch (ST_OPT_FUSED_PASSES): one thread per checkerboard pair picks the neighbour, traces the pair's two shadow
// rays and merges — the three scratch textures (48 B per pixel written and read back) never leave the registers.  Same draws, same rays
// (direction through the same octahedral round trip), same merge as the three-launch sequence.
__global__ void ST_LB_DI_SPATIAL_PICK k_di_spatial_fused(KPARAMS, int cur, u32 seed_pick, u32 seed_sample, u32 frame) {
    ST_TRACE_STACK();
    Px g = pixel_half(cam);
    if (!g.in) return;
    PairTexels o = di_spatial_pick_pair(cam, sc, cur, seed_pick, frame, g);
    if (o.state == 0) return;
    float4 d2a, d2b; trace_pair_texels(cam, sc, stk, o, g, &d2a, &d2b);
    di_spatial_sample_pair(cam, seed_sample, frame, g, d2a, d2b);
}

// K10 di_resolving::main (di_resolving.rs:4-119); ENVM (st_set_environment_map, only while a map is set): sky pixels see the map
template <bool ENVM>
__global__ void ST_LB_DI_RESOLVING k_di_resolving(KPARAMS, int cur, const __grid_constant__ EnvMapDev em) {
    ST_TRACE_STACK();
    Px p = pixel_full(cam);
    if (!p.in) return;
    size_t idx = screen_idx(cam, p.x, p.y);
    Hit hit = load_hit_lut(sc, cam.curr, cam.prim_gbuffer_d0[cur], cam.prim_gbuffer_d1[cur], cam, p.x, p.y);
    DiRes res = di_load(cam.di_reservoirs[2], idx);
    float confidence;
    LightRad rad;
    if (hit_some(hit)) {
        bool occ = trace_any(di_ray(res, hit.point), sc, stk);
        confidence = (res.occluded == occ) ? res.confidence : 0.0f;
        res.confidence = 1.0f;
        res.occluded = occ;
        if (occ) rad = lightrad_zero();
        else { rad = light_radiance(light_load(sc, res.light_id), hit); rad.radiance = rad.radiance * res.w; }
    } else {
        confidence = 1.0f;
        rad.radiance = sky_radiance<ENVM>(sc, em, world_sun_dir(sc.world), hit.dir);
        rad.diff = f3s(1.0f); rad.spec = f3s(0.0f);
    }
    float diff_brdf = (1.0f - hit.g.metallic) / kPi;
    size_t i = pix(cam, p.x, p.y);
    cam.di_diff_samples[i] = f4(rad.radiance * diff_brdf, confidence);
    cam.di_spec_samples[i] = f4(rad.radiance * rad.spec, confidence);
    di_store(res, cam.di_reservoirs[0], idx);
}

// K11 gi_reprojection::main (gi_reprojection.rs:4-51)
ST_DEV GiRes gi_reprojection_px(const CameraDev& cam, const Hit& hit, const Reproj& rp) {
    size_t npx = (size_t)cam.w * cam.h;
    GiRes res = gi_zero();
    if (reproj_some(rp)) {
        uint2 rpos = reproj_round(rp);
        size_t ridx = screen_idx(cam, rpos.x, rpos.y);
        if (ridx < npx) res = gi_load(cam.gi_reservoirs[0], ridx);
    }
    res.confidence = 1.0f;
    res.v1 = hit.point;
    return res;
}
__global__ void __launch_bounds__(ST_BLOCK) k_gi_reprojection(KPARAMS, int cur) {
    Px p = pixel_full(cam);
    if (!p.in) return;
    Hit hit = load_hit_lut(sc, cam.curr, cam.prim_gbuffer_d0[cur], cam.prim_gbuffer_d1[cur], cam, p.x, p.y);
    if (!hit_some(hit)) return;
    // strips: the columns the checkerboard passes do not cover (widths whose (W + 7) / 8 is odd) keep this entry as the spatial pass's
    // output, so there it is one of the rows a neighbouring strip's preview pass gathers
    gi_store_m(cam, gi_reprojection_px(cam, hit, reproj_decode(cam.reprojection_map[pix(cam, p.x, p.y)])), cam.gi_reservoirs[2], screen_idx(cam, p.x, p.y), p.y,
               (int)p.x >= 2 * half_grid_w(cam.w) ? cam.gi_mirror_reach : 0);
}

// K12 gi_sampling_a::main (gi_sampling_a.rs:4-122)
// returns false where the kernel leaves without writing its three scratch texels (gi_d0: ray direction + pdf, gi_d1/gi_d2: the packed
// G-buffer entry of what the ray hit)
// TEXF: the bounce hit's textures are filtered, with a fresh cone from the segment's origin
// ENVM == ENV_SAMPLED (ST_OPT_ENVIRONMENT_MAP_SAMPLING): on tracing frames one extra draw first picks, with probability 1/2, a direction
// from the map's distribution, else the BRDF's (its draws unchanged); gi_d0.w is then q / kappa (env_mixture_pdf) in place of the pdf
template <bool NMAP, bool TEXF, int ENVM>
ST_DEV bool gi_sampling_a_pair(const CameraDev& cam, const SceneDev& sc, const TraceStack& stk, int cur, u32 seed, u32 frame, Px g, float4* t0, float4* t1, float4* t2,
                               const TexFilterDev& tf, const EnvMapDev& em) {
    bool tracing = gi_tracing_frame(frame);
    uint2 sp = tracing ? checker(g.x, g.y, frame / 2u) : checker(g.x, g.y, frame);
    if (!cam_contains_u(cam.curr, sp.x, sp.y)) return false;
    size_t idx = screen_idx(cam, sp.x, sp.y);
    Ray gi_r; float gi_pdf_;
    if (tracing) {
        Rng rng = rng_make(seed, sp.x, sp.y);
        Hit hit = load_hit_lut(sc, cam.curr, cam.prim_gbuffer_d0[cur], cam.prim_gbuffer_d1[cur], cam, sp.x, sp.y);
        if (!hit_some(hit)) return false;
        if (ENVM == ENV_SAMPLED) {
            float3 dir;
            if (rng_f(rng) < 0.5f) { const float xi1 = rng_f(rng), xi2 = rng_f(rng); dir = env_draw(em, xi1, xi2); }
            else dir = brdf_layered_sample(hit.g, rng, -hit.dir).dir;
            gi_r = ray_make(hit.point, dir);
            gi_pdf_ = env_mixture_pdf(em, hit.g, -hit.dir, dir);
        } else {
            BrdfS s = brdf_layered_sample(hit.g, rng, -hit.dir);
            gi_r = ray_make(hit.point, s.dir);
            gi_pdf_ = s.pdf;
        }
    } else {
        GiRes res = gi_load(cam.gi_reservoirs[2], idx);
        if (res.m == 0.0f) return false;
        gi_r = ray_make(res.v1, gi_dir(res, res.v1));
        gi_pdf_ = 1.0f;
    }
    TriHit gh = trace_closest(gi_r, sc, stk);
    GBuf gg = gbuf_zero();
    u32 gi_color_bits = 0u;
    if (trihit_some(gh)) {
        GpuMaterial m = sc.materials[gh.material_id];
        m.roughness = rmax(m.roughness, 0.75f * 0.75f);   // Material::regularize (material.rs:25-27)
        if (TEXF) {
            TexFoot ft; ft.tri = gh.triangle_id; ft.dir = gi_r.d; ft.w = texf_cone_width(cam.curr, sp.x, sp.y, gh.t, false);
            gg.base_color = texf_sample(sc, tf, gh.material_id, 0u, m.base_color_texture, m.base_color, gh.uv, ft);
            gg.emissive = xyz(texf_sample(sc, tf, gh.material_id, 1u, m.emissive_texture, m.emissive, gh.uv, ft));
            gg.normal = NMAP ? nmap_normal(sc, gh, m.normal_map_texture) : gh.normal; gg.metallic = m.metallic;
        } else {
            gg.base_color = mat_base_color(sc, m, gh.uv); gg.normal = NMAP ? nmap_normal(sc, gh, m.normal_map_texture) : gh.normal; gg.metallic = m.metallic; gg.emissive = mat_emissive(sc, m, gh.uv);
        }
        gi_color_bits = all_zero(m.base_color_texture) ? __ldg(sc.material_packed + gh.material_id) : gbuf_pack_color(gg.base_color);
        gg.roughness = m.roughness; gg.reflectance = m.reflectance; gg.depth = dist(gi_r.o, gh.point);
    }
    gbuf_pack_pre(gg, gi_color_bits, t1, t2);
    *t0 = f4(gi_r.d, gi_pdf_);
    return true;
}
template <bool NMAP, bool TEXF, int ENVM>
__global__ void ST_LB_GI_SAMPLING_A k_gi_sampling_a(KPARAMS, int cur, u32 seed, u32 frame, const __grid_constant__ TexFilterDev tf, const __grid_constant__ EnvMapDev em) {
    ST_TRACE_STACK();
    Px g = pixel_half(cam);
    if (!g.in) return;
    float4 t0, t1, t2;
    if (!gi_sampling_a_pair<NMAP, TEXF, ENVM>(cam, sc, stk, cur, seed, frame, g, &t0, &t1, &t2, tf, em)) return;
    size_t gi = pix(cam, g.x, g.y);
    cam.gi_d0[gi] = t0; cam.gi_d1[gi] = t1; cam.gi_d2[gi] = t2;
}

// K13 gi_sampling_b::main (gi_sampling_b.rs:4-235); LGRID: the light candidates come from the light grid's list for the bounce hit
// (the sky-or-light draw still tests the global light count, so the RNG sequence keeps its shape); ENVM: the missed bounce and the sky
// draw see the map, and the sky draw's probability is 0.25 whatever the sun's altitude (the map does not darken with the sun);
// ENVM == ENV_SAMPLED: the sky draw takes its direction from the map's distribution with the same two draws, and its value is
// L max(n.w, 0) / (2 pi p_env) (no shadow ray where n.w <= 0)
template <bool LGRID, int ENVM>
ST_DEV void gi_sampling_b_pair(const CameraDev& cam, const SceneDev& sc, const TraceStack& stk, int cur, u32 seed, u32 frame, Px g, float4 d0, float4 d1, float4 d2, const LightGridDev& lg,
                               const EnvMapDev& em) {
    bool tracing = gi_tracing_frame(frame);
    uint2 sp = tracing ? checker(g.x, g.y, frame / 2u) : checker(g.x, g.y, frame);
    if (!cam_contains_u(cam.curr, sp.x, sp.y)) return;
    size_t idx = screen_idx(cam, sp.x, sp.y);
    Hit prim = load_hit_lut(sc, cam.curr, cam.prim_gbuffer_d0[cur], cam.prim_gbuffer_d1[cur], cam, sp.x, sp.y);
    if (!hit_some(prim)) return;
    Rng rng; Hit gh; float gi_pdf_;
    if (tracing) {
        rng = rng_make(seed, sp.x, sp.y);
        gh = hit_make(ray_make(prim.point, xyz(d0)), gbuf_unpack(sc, d1, d2));
        gi_pdf_ = d0.w;
    } else {
        GiRes res = gi_load(cam.gi_reservoirs[2], idx);
        if (res.m == 0.0f) return;
        rng.s = res.rng;
        gh = hit_make(ray_make(res.v1, xyz(d0)), gbuf_unpack(sc, d1, d2));
        gi_pdf_ = 1.0f;
    }
    u32 rng_state = rng.s;
    const u32 SKY = 0xffffffffu;
    float3 sun_dir = world_sun_dir(sc.world);
    u32 light_id; float light_pdf; float3 light_rad; float3 light_dir = f3s(0.f);
    bool sky_below = false;   // ENV_SAMPLED: the sky draw points below the bounce hit's surface
    if (!hit_some(gh)) { light_id = SKY; light_pdf = 1.0f; light_rad = sky_radiance<ENVM != ENV_NONE>(sc, em, sun_dir, gh.dir); }
    else {
        float atm_pdf = (ENVM == ENV_NONE && sc.world.sun_altitude <= -1.0f) ? 0.0f : 0.25f;
        if (sc.world.light_count == 0u || rng_f(rng) < atm_pdf) {
            light_id = SKY; light_pdf = atm_pdf;
            if (ENVM == ENV_SAMPLED) {
                const float xi1 = rng_f(rng), xi2 = rng_f(rng);
                light_dir = env_draw(em, xi1, xi2);
                const float c = xdot(gh.g.normal, light_dir);
                sky_below = !(c > 0.0f);
                const float p = sky_below ? 0.0f : env_pdf(em, light_dir);
                light_rad = p > 0.0f ? xscale(env_sample(em, light_dir), xdiv(c, xmul(6.283185307179586f, p))) : f3s(0.0f);
            } else {
                light_dir = rng_hemisphere(rng, gh.g.normal);
                light_rad = sky_radiance<ENVM != ENV_NONE>(sc, em, sun_dir, light_dir) * dot(gh.g.normal, light_dir);
            }
        } else {
            EphRes er = LGRID ? ephemeral_build_list(rng, sc, gh, lgrid_list(lg, gh.point)) : ephemeral_build(rng, sc, gh);
            if (er.w > 0.0f) { light_id = er.light_id; light_pdf = (1.0f / er.w) * (1.0f - atm_pdf); light_rad = er.rad.radiance * (f3s(1.0f) + er.rad.spec); }
            else { light_id = 0u; light_pdf = 1.0f; light_rad = f3s(0.f); }
        }
    }
    float3 radiance;
    if (light_pdf > 0.0f) {
        float vis;
        if (hit_some(gh)) {
            if (ENVM == ENV_SAMPLED && sky_below) vis = 0.0f;
            else {
                Ray r = (light_id == SKY) ? ray_make(gh.point, light_dir) : light_ray_wnoise(light_load(sc, light_id), rng, gh.point);
                vis = trace_any(r, sc, stk) ? 0.0f : 1.0f;
            }
        } else vis = 1.0f;
        radiance = light_rad * vis / light_pdf;
    } else radiance = f3s(0.f);
    if (hit_some(gh)) { radiance = radiance * (xyz(gh.g.base_color) / kPi); radiance = radiance + gh.g.emissive; }
    GiRes res = gi_zero();
    if (gi_pdf_ > 0.0f) {
        res.rng = rng_state; res.radiance = radiance; res.v1 = prim.point;
        if (hit_some(gh)) { res.v2 = gh.point; res.v2n = gh.g.normal; }
        else { res.v2 = prim.point + gh.dir * 1000.0f; res.v2n = -gh.dir; }
        res.m = 1.0f; res.w = 1.0f / gi_pdf_;
        res.pdf = 0.0f;
        res.pdf = gi_pdf(res, prim);
    }
    gi_store(res, cam.gi_reservoirs[1], idx);
}
template <bool LGRID, int ENVM>
__global__ void ST_LB_GI_SAMPLING_B k_gi_sampling_b(KPARAMS, int cur, u32 seed, u32 frame, const __grid_constant__ LightGridDev lg, const __grid_constant__ EnvMapDev em) {
    ST_TRACE_STACK();
    Px g = pixel_half(cam);
    if (!g.in) return;
    size_t gi = pix(cam, g.x, g.y);
    gi_sampling_b_pair<LGRID, ENVM>(cam, sc, stk, cur, seed, frame, g, cam.gi_d0[gi], cam.gi_d1[gi], cam.gi_d2[gi], lg, em);
}
// K12 + K13 in one launch (ST_OPT_FUSED_PASSES): the bounce ray is traced and shaded by the same thread; the hit still goes through
// GBufferEntry's pack / unpack (its 8-bit quantisation is part of the result), just not through memory.
template <bool NMAP, bool LGRID, bool TEXF, int ENVM>
__global__ void ST_LB_GI_SAMPLING_B k_gi_sampling_fused(KPARAMS, int cur, u32 seed_a, u32 seed_b, u32 frame, const __grid_constant__ LightGridDev lg,
                                                        const __grid_constant__ TexFilterDev tf, const __grid_constant__ EnvMapDev em) {
    ST_TRACE_STACK();
    Px g = pixel_half(cam);
    if (!g.in) return;
    float4 t0, t1, t2;
    if (!gi_sampling_a_pair<NMAP, TEXF, ENVM == ENV_SAMPLED ? ENV_SAMPLED : ENV_NONE>(cam, sc, stk, cur, seed_a, frame, g, &t0, &t1, &t2, tf, em)) return;
    gi_sampling_b_pair<LGRID, ENVM>(cam, sc, stk, cur, seed_b, frame, g, t0, t1, t2, lg, em);
}

// K14 gi_temporal_resampling::main (gi_temporal_resampling.rs:4-156)
// `inline_reprojection` (ST_OPT_FUSED_PASSES, tracing frames): K11 is evaluated here instead of in its own launch — last frame's
// reservoir is fetched from gi_reservoirs[0] at the reprojected position directly, and handed on as K11 would have left it in
// gi_reservoirs[2] (its normal goes through the same octahedral store / load round trip).  gi_reservoirs[2] itself is then only written
// for the columns a later pass still reads there (those the checkerboard passes do not cover when the width is odd).
__global__ void ST_LB_GI_TEMPORAL k_gi_temporal(KPARAMS, int cur, u32 seed, u32 frame, int inline_reprojection) {
    Px p = pixel_full(cam);
    if (!p.in) return;
    bool tracing = gi_tracing_frame(frame);
    size_t lhs_idx = screen_idx(cam, p.x, p.y);
    Rng rng = rng_make(seed, p.x, p.y);
    Hit lhs_hit = load_hit_lut(sc, cam.curr, cam.prim_gbuffer_d0[cur], cam.prim_gbuffer_d1[cur], cam, p.x, p.y);
    float4* curr = cam.gi_reservoirs[1];
    if (!hit_some(lhs_hit)) { gi_store_m(cam, gi_zero(), curr, lhs_idx, p.y, cam.gi_mirror_reach); return; }
    bool got = tracing ? (frame % 2u == 0u && checker_at(p.x, p.y, frame / 2u)) : checker_at(p.x, p.y, frame);
    GiRes lhs = got ? gi_load(curr, lhs_idx) : gi_zero();
    GiRes rhs = gi_zero();
    Hit rhs_hit = hit_zero();
    Reproj rp = reproj_decode(cam.reprojection_map[pix(cam, p.x, p.y)]);
    if (inline_reprojection) {
        GiRes r11 = gi_reprojection_px(cam, lhs_hit, rp);
        if ((int)p.x >= 2 * half_grid_w(cam.w)) gi_store_m(cam, r11, cam.gi_reservoirs[2], lhs_idx, p.y, cam.gi_mirror_reach);
        if (reproj_some(rp)) { rhs = r11; rhs.v2n = oct_decode(oct_encode(r11.v2n)); }
    } else if (reproj_some(rp)) rhs = gi_load(cam.gi_reservoirs[2], lhs_idx);
    if (reproj_some(rp)) {
        rhs.confidence = 1.0f;
        rhs.m = rmin(rhs.m, 128.0f);
        if (!tracing && lhs.m != 0.0f && rhs.m != 0.0f && gi_exists(rhs)) {
            if (dist(lhs.radiance, rhs.radiance) > 0.33f) rhs.confidence = 0.0f;
            rhs.radiance = lhs.radiance; rhs.v2 = lhs.v2; rhs.v2n = lhs.v2n;
        }
        if (rhs.m != 0.0f) {
            uint2 rpos = reproj_round(rp);
            rhs_hit = load_hit_lut(sc, cam.prev, cam.prim_gbuffer_d0[cur ^ 1], cam.prim_gbuffer_d1[cur ^ 1], cam, rpos.x, rpos.y);
        }
    }
    GiRes main_ = gi_zero();
    float main_pdf = 0.0f;
    if (tracing) {
        MisIn mi;
        mi.lhs_m = lhs.m; mi.rhs_m = rhs.m; mi.rhs_jacobian = 1.0f; mi.lhs_lhs_pdf = lhs.pdf; mi.rhs_rhs_pdf = rhs.pdf;
        mi.lhs_rhs_pdf = ((lhs.m > 0.0f) & hit_some(rhs_hit)) ? gi_pdf(lhs, rhs_hit) : 0.0f;
        mi.rhs_lhs_pdf = (rhs.m > 0.0f) ? gi_pdf(rhs, lhs_hit) : 0.0f;
        MisOut mo = mis_eval(mi);
        if (gi_update(main_, rng, lhs, mo.lhs_mis * mo.lhs_pdf * lhs.w)) main_pdf = mo.lhs_pdf;
        if (gi_update(main_, rng, rhs, mo.rhs_mis * mo.rhs_pdf * rhs.w)) main_pdf = mo.rhs_pdf;
        main_.m = lhs.m + mo.m;
        main_.confidence = 1.0f;
        main_.w = res_norm(main_.w, main_pdf, 1.0f, 1.0f);
    } else {
        if (gi_merge(main_, rng, rhs, rhs.pdf)) main_pdf = rhs.pdf;
        main_.confidence = rhs.confidence;
        main_.w = res_norm(main_.w, main_pdf, 1.0f, main_.m);
    }
    main_.pdf = main_pdf;
    main_.v1 = lhs_hit.point;
    main_.w = rmin(main_.w, 5.0f);
    gi_store_m(cam, main_, curr, lhs_idx, p.y, cam.gi_mirror_reach);
}

// K15 gi_spatial_resampling::pick (gi_spatial_resampling.rs:4-160); scratch = gi_d0, gi_d1
ST_DEV PairTexels gi_spatial_pick_pair(const CameraDev& cam, const SceneDev& sc, int cur, u32 seed, u32 frame, Px g) {
    PairTexels o; o.a0 = o.a1 = o.b0 = o.b1 = f4zero(); o.state = 0;
    uint2 lp = checker(g.x, g.y, frame / 2u + 1u);
    if (!cam_contains_u(cam.curr, lp.x, lp.y)) return o;
    o.state = 1;
    size_t lhs_idx = screen_idx(cam, lp.x, lp.y);
    Rng rng = rng_make(seed, lp.x, lp.y);
    const float4* gd0 = cam.prim_gbuffer_d0[cur]; const float4* gd1 = cam.prim_gbuffer_d1[cur];
    const float4* reservoirs = cam.gi_reservoirs[1];
    Hit lhs_hit = load_hit_lut(sc, cam.curr, gd0, gd1, cam, lp.x, lp.y);
    GiRes lhs = gi_load(reservoirs, lhs_idx);
    if (!hit_some(lhs_hit) || lhs.m == 0.0f) return o;
    GiRes rhs = gi_zero();
    size_t rhs_idx = 0;
    Hit rhs_hit = hit_zero();
    float rhs_jac = 0.0f;
    float max_radius = 128.0f;
    for (u32 nth = 0u; nth < 8u; nth++) {
        float2 off = rng_disk(rng) * max_radius;
        float2 fp = f2((float)lp.x, (float)lp.y) + off;
        uint2 rpos = cam_contain(cam.curr, to_i32_sat(fp.x), to_i32_sat(fp.y));
        if (rpos.x == lp.x && rpos.y == lp.y) continue;
        float4 nd = tex_or_zero(cam.surface_nd, cam, rpos.x, rpos.y);
        if (nd.w == 0.0f) { max_radius = rmax(max_radius * 0.5f, 5.0f); continue; }
        if (fabs_(nd.w - lhs_hit.g.depth) > 0.33f * lhs_hit.g.depth) { max_radius = rmax(max_radius * 0.5f, 5.0f); continue; }
        if (dot(xyz(nd), lhs_hit.g.normal) < 0.33f) { max_radius = rmax(max_radius * 0.5f, 5.0f); continue; }
        rhs_idx = screen_idx(cam, rpos.x, rpos.y);
        rhs = gi_load(reservoirs, rhs_idx);
        if (rhs.m == 0.0f) continue;
        rhs_jac = gi_jacobian(rhs, lhs_hit.point);
        if (rhs_jac < 1.0f / 10.0f || rhs_jac > 10.0f) { rhs.m = 0.0f; continue; }
        rhs_jac = rclamp(rhs_jac, 1.0f / 3.0f, 3.0f);
        rhs_hit = load_hit_lut(sc, cam.curr, gd0, gd1, cam, rpos.x, rpos.y);
        break;
    }
    if (rhs.m == 0.0f || !hit_some(rhs_hit)) return o;
    float lhs_rhs_pdf = gi_pdf(lhs, rhs_hit);
    float rhs_lhs_pdf = gi_pdf(rhs, lhs_hit);
    Ray ra = (lhs_rhs_pdf > 0.0f) ? gi_ray(lhs, rhs_hit.point) : ray_zero();
    Ray rb = (rhs_lhs_pdf > 0.0f) ? gi_ray(rhs, lhs_hit.point) : ray_zero();
    float2 na = oct_encode(ra.d), nb = oct_encode(rb.d);
    o.a0 = f4(ra.o, ra.len); o.a1 = f4(na.x, na.y, bitsf((u32)rhs_idx + 1u), rhs_jac);
    o.b0 = f4(rb.o, rb.len); o.b1 = f4(nb.x, nb.y, lhs_rhs_pdf, rhs_lhs_pdf);
    o.state = 2;
    return o;
}
__global__ void ST_LB_GI_SPATIAL_PICK k_gi_spatial_pick(KPARAMS, int cur, u32 seed, u32 frame) {
    Px g = pixel_half(cam);
    if (!g.in) return;
    store_pair_texels(cam, gi_spatial_pick_pair(cam, sc, cur, seed, frame, g), cam.gi_d0, cam.gi_d1, g);
}

// K17 gi_spatial_resampling::sample (gi_spatial_resampling.rs:225-314)
ST_DEV void gi_spatial_sample_pair(const CameraDev& cam, u32 seed, u32 frame, Px g, float4 d0, float4 d1) {
    uint2 sp = checker(g.x, g.y, frame / 2u + 1u);
    if (!cam_contains_u(cam.curr, sp.x, sp.y)) return;
    size_t npx = (size_t)cam.w * cam.h;
    size_t idx = screen_idx(cam, sp.x, sp.y);
    Rng rng = rng_make(seed, sp.x, sp.y);
    const float4* in = cam.gi_reservoirs[1]; float4* out = cam.gi_reservoirs[2];
    float lhs_rhs_vis = d0.x; u32 rhs_idx = fbits(d0.y); float rhs_jac = d0.z;
    float rhs_lhs_vis = d1.x, lhs_rhs_pdf = d1.y, rhs_lhs_pdf = d1.z;
    GiRes lhs = gi_load(in, idx);
    if (rhs_idx > 0u && (size_t)rhs_idx - 1 < npx) {
        GiRes rhs = gi_load(in, (size_t)rhs_idx - 1);
        MisIn mi;
        mi.lhs_m = lhs.m; mi.rhs_m = rhs.m; mi.rhs_jacobian = rhs_jac; mi.lhs_lhs_pdf = lhs.pdf;
        mi.lhs_rhs_pdf = lhs_rhs_pdf * lhs_rhs_vis; mi.rhs_lhs_pdf = rhs_lhs_pdf * rhs_lhs_vis; mi.rhs_rhs_pdf = rhs.pdf;
        MisOut mo = mis_eval(mi);
        GiRes main_ = gi_zero();
        float main_pdf = 0.0f;
        if (gi_update(main_, rng, lhs, mo.lhs_mis * mo.lhs_pdf * lhs.w)) main_pdf = mo.lhs_pdf;
        if (gi_update(main_, rng, rhs, mo.rhs_mis * mo.rhs_pdf * rhs.w * rhs_jac)) main_pdf = mo.rhs_pdf;
        main_.m = lhs.m + mo.m;
        main_.confidence = 1.0f;
        main_.pdf = main_pdf;
        main_.v1 = lhs.v1;
        main_.w = res_norm(main_.w, main_pdf, 1.0f, 1.0f);
        main_.w = rmin(main_.w, 5.0f);
        gi_store_m(cam, main_, out, idx, sp.y, cam.gi_mirror_reach);
    } else gi_store_m(cam, lhs, out, idx, sp.y, cam.gi_mirror_reach);
    uint2 op = checker(g.x, g.y, frame / 2u);
    if (cam_contains_u(cam.curr, op.x, op.y)) { size_t oi = screen_idx(cam, op.x, op.y); gi_store_m(cam, gi_load(in, oi), out, oi, op.y, cam.gi_mirror_reach); }
}
__global__ void ST_LB_GI_SPATIAL_SAMPLE k_gi_spatial_sample(KPARAMS, u32 seed, u32 frame) {
    Px g = pixel_half(cam);
    if (!g.in) return;
    gi_spatial_sample_pair(cam, seed, frame, g, tex_or_zero(cam.gi_d2, cam, g.x * 2u, g.y), tex_or_zero(cam.gi_d2, cam, g.x * 2u + 1u, g.y));
}
// K15 + K16 + K17 in one launch (ST_OPT_FUSED_PASSES), like k_di_spatial_fused
__global__ void ST_LB_GI_SPATIAL_PICK k_gi_spatial_fused(KPARAMS, int cur, u32 seed_pick, u32 seed_sample, u32 frame) {
    ST_TRACE_STACK();
    Px g = pixel_half(cam);
    if (!g.in) return;
    PairTexels o = gi_spatial_pick_pair(cam, sc, cur, seed_pick, frame, g);
    if (o.state == 0) return;
    float4 d2a, d2b; trace_pair_texels(cam, sc, stk, o, g, &d2a, &d2b);
    gi_spatial_sample_pair(cam, seed_sample, frame, g, d2a, d2b);
}

// K18 gi_preview_resampling::main (gi_preview_resampling.rs:4-138).  Returns false where the kernel exits without writing (quirk C-6).
ST_DEV bool gi_preview_px(const CameraDev& cam, const SceneDev& sc, const Hit& chit, u32 seed, u32 nth, const float4* __restrict__ in, Px p, GiRes* result) {
    size_t cidx = screen_idx(cam, p.x, p.y);
    Rng rng = rng_make(seed, p.x, p.y);
    if (!hit_some(chit)) { *result = gi_zero(); return true; }
    GiRes main_ = gi_zero();
    float main_pdf = 0.0f;
    GiRes center = gi_load(in, cidx);
    if (gi_merge(main_, rng, center, center.pdf)) main_pdf = center.pdf;
    u32 max_samples = to_u32_sat(lerpc(8.0f, 0.0f, main_.m / 8.0f));
    float max_radius = (nth == 0u) ? 128.0f : 64.0f;
    const float4* __restrict__ surf = cam.surface_nd;
    for (u32 k = 0u; k < max_samples; k++) {
        float2 off = rng_disk(rng) * max_radius;
        float2 fp = f2((float)p.x, (float)p.y) + off;
        uint2 sp = cam_contain(cam.curr, to_i32_sat(fp.x), to_i32_sat(fp.y));
        if (sp.x == p.x && sp.y == p.y) return false;   // quirk C-6: the kernel exits without writing
        if (!cam_contains_u(cam.curr, sp.x, sp.y)) continue;
        float4 nd = surf[pix(cam, sp.x, sp.y)];
        if (nd.w == 0.0f) continue;
        if (fabs_(nd.w - chit.g.depth) > 0.25f * chit.g.depth) continue;
        if (dot(xyz(nd), chit.g.normal) < 0.5f) continue;
        GiRes s = gi_load(in, screen_idx(cam, sp.x, sp.y));
        if (s.m == 0.0f) continue;
        float s_pdf = gi_pdf(s, chit);
        float s_jac = gi_jacobian(s, chit.point);
        if (s_jac < 1.0f / 10.0f || s_jac > 10.0f) continue;
        s_jac = rclamp(s_jac, 1.0f / 3.0f, 3.0f);
        if (gi_merge(main_, rng, s, s_pdf * s_jac)) main_pdf = s_pdf;
    }
    main_.confidence = center.confidence;
    main_.pdf = main_pdf;
    main_.v1 = center.v1;
    main_.w = res_norm(main_.w, main_pdf, 1.0f, main_.m);
    main_.w = rmin(main_.w, 5.0f);
    *result = main_;
    return true;
}
__global__ void ST_LB_GI_PREVIEW k_gi_preview(KPARAMS, int cur, u32 seed, u32 nth, const float4* __restrict__ in, float4* __restrict__ out, int reach) {
    Px p = pixel_full(cam);
    if (!p.in) return;
    Hit chit = load_hit_lut(sc, cam.curr, cam.prim_gbuffer_d0[cur], cam.prim_gbuffer_d1[cur], cam, p.x, p.y);
    GiRes r;
    if (gi_preview_px(cam, sc, chit, seed, nth, in, p, &r)) gi_store_m(cam, r, out, screen_idx(cam, p.x, p.y), p.y, reach);
}

// K19 gi_resolving::main (gi_resolving.rs:4-67): shades the pixel from `res` (the entry the second preview pass left in gi_reservoirs[0]),
// then replaces that entry with the frame's source reservoir
ST_DEV void gi_resolving_px(const CameraDev& cam, const Hit& hit, const GiRes& res, const float4* __restrict__ in, Px p) {
    size_t idx = screen_idx(cam, p.x, p.y);
    float confidence; float3 radiance;
    if (hit_some(hit)) { confidence = res.confidence; radiance = res.w * gi_cosine(res, hit) * res.radiance; }
    else { confidence = 1.0f; radiance = f3s(0.f); }
    float diff_brdf = (1.0f - hit.g.metallic) / kPi;
    float3 spec = gi_spec(res, hit);
    size_t i = pix(cam, p.x, p.y);
    cam.gi_diff_samples[i] = f4(radiance * diff_brdf, confidence);
    cam.gi_spec_samples[i] = f4(radiance * spec, confidence);
    gi_store(gi_load(in, idx), cam.gi_reservoirs[0], idx);
}
__global__ void ST_LB_GI_RESOLVING k_gi_resolving(KPARAMS, int cur, const float4* __restrict__ in) {
    Px p = pixel_full(cam);
    if (!p.in) return;
    Hit hit = load_hit_lut(sc, cam.curr, cam.prim_gbuffer_d0[cur], cam.prim_gbuffer_d1[cur], cam, p.x, p.y);
    gi_resolving_px(cam, hit, gi_load(cam.gi_reservoirs[0], screen_idx(cam, p.x, p.y)), in, p);
}
// second preview pass + K19 in one launch (ST_OPT_FUSED_PASSES): the pass's result is shaded straight away instead of going through
// gi_reservoirs[0] (K19 only consumes fields that a store / load leaves untouched); where the pass exits without writing (quirk C-6) K19
// sees last frame's entry, which is what is loaded here then.
__global__ void ST_LB_GI_PREVIEW k_gi_preview_resolve(KPARAMS, int cur, u32 seed, const float4* __restrict__ in, const float4* __restrict__ source) {
    Px p = pixel_full(cam);
    if (!p.in) return;
    Hit chit = load_hit_lut(sc, cam.curr, cam.prim_gbuffer_d0[cur], cam.prim_gbuffer_d1[cur], cam, p.x, p.y);
    GiRes r;
    if (!gi_preview_px(cam, sc, chit, seed, 1u, in, p, &r)) r = gi_load(cam.gi_reservoirs[0], screen_idx(cam, p.x, p.y));
    gi_resolving_px(cam, chit, r, source, p);
}

#if ST_EXACT_ONLY
// K20 frame_denoising::reproject (frame_denoising.rs:4-78)
__global__ void __launch_bounds__(ST_BLOCK) k_denoise_reproject(KPARAMS, int cur, const float4* __restrict__ prev_colors, const float4* __restrict__ prev_moments,
                                                                const float4* __restrict__ samples, float4* __restrict__ colors, float4* __restrict__ moments) {
    Px p = pixel_full(cam);
    if (!p.in) return;
    size_t i = pix(cam, p.x, p.y);
    float4 sample = samples[i];
    if (cam.prim_surface_map[cur][i].z == 0.0f) { store4m(cam, colors + i, sample, p.y, ST_REACH_SVGF); return; }
    float sl = luma(xyz(sample));
    Reproj rp = reproj_decode(cam.reprojection_map[i]);
    float3 color, moment;
    if (reproj_some(rp) && sample.w > 0.0f) {
        float4 pc = history_fetch(rp, prev_colors, cam.w, cam.h);
        float4 pm = history_fetch(rp, prev_moments, cam.w, cam.h);
        float hist = rmin(pm.x + 1.0f, 16.0f);
        float alpha = 1.0f / hist;
        color = lerpc(xyz(pc), xyz(sample), alpha);
        moment = f3(hist, lerpc(pm.y, sl, alpha), lerpc(pm.z, sl * sl, alpha));
    } else { color = xyz(sample); moment = f3(1.0f, sl, sl * sl); }
    store4m(cam, colors + i, f4(color, 0.0f), p.y, ST_REACH_SVGF);
    store4m(cam, moments + i, f4(moment, 0.0f), p.y, ST_REACH_SVGF);
}

// K20 for the DI and the GI signal in one launch: the surface depth and the reprojection entry are read once
// (192 instead of 2 x 112 B/px); per signal exactly the arithmetic of k_denoise_reproject.
struct ReprojectSignal { const float4* prev_colors; const float4* prev_moments; const float4* samples; float4* colors; float4* moments; };
ST_DEV void denoise_reproject_signal(const CameraDev& cam, size_t i, u32 y, float4 sample, const Reproj& rp, bool has_rp, const ReprojectSignal& g) {
    float sl = luma(xyz(sample));
    float3 color, moment;
    if (has_rp && sample.w > 0.0f) {
        float4 pc = history_fetch(rp, g.prev_colors, cam.w, cam.h);
        float4 pm = history_fetch(rp, g.prev_moments, cam.w, cam.h);
        float hist = rmin(pm.x + 1.0f, 16.0f);
        float alpha = 1.0f / hist;
        color = lerpc(xyz(pc), xyz(sample), alpha);
        moment = f3(hist, lerpc(pm.y, sl, alpha), lerpc(pm.z, sl * sl, alpha));
    } else { color = xyz(sample); moment = f3(1.0f, sl, sl * sl); }
    store4m(cam, g.colors + i, f4(color, 0.0f), y, ST_REACH_SVGF);
    store4m(cam, g.moments + i, f4(moment, 0.0f), y, ST_REACH_SVGF);
}
__global__ void __launch_bounds__(ST_BLOCK) k_denoise_reproject_pair(KPARAMS, int cur, const __grid_constant__ ReprojectSignal di, const __grid_constant__ ReprojectSignal gi) {
    Px p = pixel_full(cam);
    if (!p.in) return;
    size_t i = pix(cam, p.x, p.y);
    float4 sd = di.samples[i], sg = gi.samples[i];
    if (cam.prim_surface_map[cur][i].z == 0.0f) { store4m(cam, di.colors + i, sd, p.y, ST_REACH_SVGF); store4m(cam, gi.colors + i, sg, p.y, ST_REACH_SVGF); return; }
    Reproj rp = reproj_decode(cam.reprojection_map[i]);
    bool has_rp = reproj_some(rp);
    denoise_reproject_signal(cam, i, p.y, sd, rp, has_rp, di);
    denoise_reproject_signal(cam, i, p.y, sg, rp, has_rp, gi);
}

// frame_denoising::sample_weight (frame_denoising.rs:363-392), split into the part that is common to
// the DI and GI signals (depth ramp, normal^64) and the per-signal luminance term:
//   weight = exp(-|sqrt(lc) - sqrt(ls)| * luma_sigma) * depth_weight * normal_weight
// A zero depth or normal factor makes the product 0 (or NaN), never > 0, so the caller may skip the tap.
//
// Two arithmetic flavours (template parameter FAST):
//   FAST = false  strict IEEE f32 with the polynomial exp: bit-identical to the CPU oracle.
//   FAST = true   the SFU approximations a GPU shader compiler emits for GLSL exp/sqrt/div
//                 (ex2.approx, sqrt.approx, rcp.approx; <= 2 ulp each) and fused multiply-adds.  Only the
//                 edge-stopping weights / normalisation of the denoiser use it; reservoirs, hits and every
//                 other buffer stay bit-exact, the denoised colours stay inside north_star's 1e-3 tolerance.
ST_DEV float sfu_ex2(float x) { float r; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
ST_DEV float sfu_sqrt(float x) { float r; asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
ST_DEV float sfu_rcp(float x) { float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
template <bool FAST> ST_DEV float sv_sqrt(float x) { return FAST ? sfu_sqrt(x) : sqrtf(x); }
template <bool FAST> ST_DEV float sv_luma(float3 c) { return FAST ? __fmaf_rn(c.z, 0.0722f, __fmaf_rn(c.y, 0.7152f, c.x * 0.2126f)) : luma(c); }
template <bool FAST> ST_DEV float svgf_depth_weight(float c_depth, float s_depth, float depth_sigma) {
    float leeway = c_depth * depth_sigma;
    float diff = fabs_(s_depth - c_depth);
    if (diff >= leeway) return 0.0f;
    return FAST ? __fmaf_rn(-diff, sfu_rcp(leeway), 1.0f) : 1.0f - diff / leeway;
}
template <bool FAST> ST_DEV float svgf_normal_weight(float3 c_normal, float3 s_normal) {
    float d = FAST ? __fmaf_rn(s_normal.z, c_normal.z, __fmaf_rn(s_normal.y, c_normal.y, s_normal.x * c_normal.x)) : dot(s_normal, c_normal);
    return pow_det(rmax(d, 0.0f), 64.0f);   // six squarings
}
template <bool FAST> ST_DEV float svgf_luma_weight(float sqrt_center_luma, float sample_luma, float luma_sigma) {
    float lw = fabs_(sqrt_center_luma - sv_sqrt<FAST>(sample_luma)) * luma_sigma;
    return FAST ? sfu_ex2(lw * -1.44269504088896341f) : exp_det(-lw);
}

// K21 frame_denoising::estimate_variance (frame_denoising.rs:81-217)
template <bool FAST>
__global__ void __launch_bounds__(ST_BLOCK) k_denoise_variance(KPARAMS, int cur) {
    Px p = pixel_full(cam);
    if (!p.in) return;
    size_t i = pix(cam, p.x, p.y);
    const float4* __restrict__ snd = cam.surface_nd;
    const float4* __restrict__ di_colors = cam.di_diff_curr_colors; const float4* __restrict__ gi_colors = cam.gi_diff_curr_colors;
    float4 cnd = snd[i];
    float4 cdi = di_colors[i], cgi = gi_colors[i];
    if (cnd.w == 0.0f) { cam.di_diff_stash[i] = cdi; cam.gi_diff_stash[i] = cgi; return; }
    float4 mdi = cam.di_diff_moments[cur][i], mgi = cam.gi_diff_moments[cur][i];
    float di_var, gi_var;
    if (mdi.x >= 4.0f) { di_var = mdi.z - sq(mdi.y); gi_var = mgi.z - sq(mgi.y); }
    else {
        float3 cn = xyz(cnd);
        float scdl = sv_sqrt<FAST>(sv_luma<FAST>(xyz(cdi))), scgl = sv_sqrt<FAST>(sv_luma<FAST>(xyz(cgi)));
        float3 sdi = f3s(0.f), sgi = f3s(0.f);
        int ox = -2, oy = -2;
        for (;;) {   // quirk C-3: row -2 spans x in [-2,2], rows -1..2 span x in [-3,2]
            int sx = (int)p.x + ox, sy = (int)p.y + oy;
            if (cam_contains_i(cam.curr, sx, sy)) {
                size_t si = pix(cam, (u32)sx, (u32)sy);
                float4 nds = snd[si];
                if (nds.w != 0.0f) {
                    float common = svgf_depth_weight<FAST>(cnd.w, nds.w, 0.2f);
                    float nw = svgf_normal_weight<FAST>(cn, xyz(nds));
                    float sl = sv_luma<FAST>(xyz(di_colors[si]));
                    float w = svgf_luma_weight<FAST>(scdl, sl, 1.0f) * common * nw;
                    sdi = sdi + f3(sl, sl * sl, 1.0f) * f3s(w);
                    float gl = sv_luma<FAST>(xyz(gi_colors[si]));
                    float wg = svgf_luma_weight<FAST>(scgl, gl, 1.0f) * common * nw;
                    sgi = sgi + f3(gl, gl * gl, 1.0f) * f3s(wg);
                }
            }
            ox += 1;
            if (ox == 3) { ox = -3; oy += 1; if (oy == 3) break; }
        }
        { float m1 = sdi.x / sdi.z, m2 = sdi.y / sdi.z; di_var = fabs_(m2 - m1 * m1) * 4.0f; }
        { float m1 = sgi.x / sgi.z, m2 = sgi.y / sgi.z; gi_var = fabs_(m2 - m1 * m1) * 4.0f; }
    }
    di_var = rmax(di_var, 0.0f); gi_var = rmax(gi_var, 0.0f);
    cam.di_diff_stash[i] = f4(xyz(cdi), di_var);
    cam.gi_diff_stash[i] = f4(xyz(cgi), gi_var);
}

// K22 frame_denoising::wavelet (frame_denoising.rs:220-361): 3x3 à-trous, DI and GI together.
// Per tap: one (normal, depth) float4 + the two signal float4s; the depth ramp and normal^64 factors are
// evaluated once and shared by both signals, taps whose shared factor is 0 are skipped (weight cannot be > 0).
#ifndef ST_WAVELET_MIN_BLOCKS
#define ST_WAVELET_MIN_BLOCKS 10
#endif
// PAIR_IN: the two signals arrive interleaved, {DI, GI} = one 32-byte record per pixel (`pair_in`, written by the previous iteration
// through `pair_out`), so that a jittered tap of the wide strides is one full sector (two 128-bit loads on sm_90a) instead of two
// half-used sectors; `pair_out` != nullptr writes that layout.  Values and arithmetic are those of the planar layout.
template <bool FAST, bool PAIR_IN>
__global__ void __launch_bounds__(ST_BLOCK, ST_WAVELET_MIN_BLOCKS) k_denoise_wavelet(KPARAMS, int cur, u32 frame, u32 stride, float strength,
                                                              const float4* __restrict__ di_in, float4* __restrict__ di_out,
                                                              const float4* __restrict__ gi_in, float4* __restrict__ gi_out,
                                                              const float4* __restrict__ pair_in, float4* __restrict__ pair_out) {
    Px p = pixel_full(cam);
    if (!p.in) return;
    size_t i = pix(cam, p.x, p.y);
    const float4* __restrict__ snd = cam.surface_nd;
    float4 cnd = snd[i];
    float4 cdi, cgi;
    if (PAIR_IN) { F8 c = ld8(pair_in + 2 * i); cdi = c.a; cgi = c.b; } else cdi = di_in[i];
    float3 cdc = xyz(cdi); float cdv = cdi.w;
    if (cnd.w == 0.0f) { if (pair_out) pair_out[2 * i] = f4(cdc, cdv); else di_out[i] = f4(cdc, cdv); return; }
    float4 bn = blue_noise(sc, p.x, p.y, frame);
    if (!PAIR_IN) cgi = gi_in[i];
    float3 cgc = xyz(cgi); float cgv = cgi.w;
    float3 cn = xyz(cnd);
    float scdl = sv_sqrt<FAST>(sv_luma<FAST>(cdc)), scgl = sv_sqrt<FAST>(sv_luma<FAST>(cgc));
    float ls_di = lerpc(2.5f, 0.5f, sv_sqrt<FAST>(cdv));
    float ls_gi = lerpc(1.0f, 0.0f, sv_sqrt<FAST>(cgv));
    float depth_sigma = 0.33f / strength;   // same for DI and GI (frame_denoising.rs:264,267)
    float2 jf = (f2(bn.z, bn.w) - f2(0.5f, 0.5f)) * ((float)stride - 1.0f) * 0.5f;
    int jx = to_i32_sat(jf.x), jy = to_i32_sat(jf.y);
    float sdw = 1.0f; float3 sdc = cdc; float sdv = cdv;
    float sgw = 1.0f; float3 sgc = cgc; float sgv = cgv;
#pragma unroll
    for (int oy = -1; oy <= 1; oy++) {
#pragma unroll
        for (int ox = -1; ox <= 1; ox++) {
            if (ox == 0 && oy == 0) continue;
            int sx = (int)p.x + jx + ox * (int)stride, sy = (int)p.y + jy + oy * (int)stride;
            if (!cam_contains_i(cam.curr, sx, sy)) continue;
            size_t si = pix(cam, (u32)sx, (u32)sy);
            float4 nds = snd[si];
            if (nds.w == 0.0f) continue;
            float dw = svgf_depth_weight<FAST>(cnd.w, nds.w, depth_sigma);
            float nw = svgf_normal_weight<FAST>(cn, xyz(nds));
            if (dw == 0.0f || nw == 0.0f) continue;
            float dnw = dw * nw;
            float4 sdi, sgi;
            if (PAIR_IN) { F8 t = ld8(pair_in + 2 * si); sdi = t.a; sgi = t.b; } else { sdi = di_in[si]; sgi = gi_in[si]; }
            if (FAST) {
                float wd = svgf_luma_weight<true>(scdl, sv_luma<true>(xyz(sdi)), ls_di) * dnw;
                if (wd > 0.0f) { sdw += wd; sdc = f3(__fmaf_rn(wd, sdi.x, sdc.x), __fmaf_rn(wd, sdi.y, sdc.y), __fmaf_rn(wd, sdi.z, sdc.z)); sdv = __fmaf_rn(wd * wd, sdi.w, sdv); }
                float wg = svgf_luma_weight<true>(scgl, sv_luma<true>(xyz(sgi)), ls_gi) * dnw;
                if (wg > 0.0f) { sgw += wg; sgc = f3(__fmaf_rn(wg, sgi.x, sgc.x), __fmaf_rn(wg, sgi.y, sgc.y), __fmaf_rn(wg, sgi.z, sgc.z)); sgv = __fmaf_rn(wg * wg, sgi.w, sgv); }
            } else {
                float wd = svgf_luma_weight<false>(scdl, luma(xyz(sdi)), ls_di) * dw * nw;
                if (wd > 0.0f) { sdw += wd; sdc = sdc + wd * xyz(sdi); sdv += sq(wd) * sdi.w; }
                float wg = svgf_luma_weight<false>(scgl, luma(xyz(sgi)), ls_gi) * dw * nw;
                if (wg > 0.0f) { sgw += wg; sgc = sgc + wg * xyz(sgi); sgv += sq(wg) * sgi.w; }
            }
        }
    }
    float4 odi, ogi;
    if (FAST) {
        float rd = sfu_rcp(sdw), rg = sfu_rcp(sgw);
        odi = f4(sdc * rd, sdv * (rd * rd));
        ogi = f4(sgc * rg, sgv * (rg * rg));
    } else {
        odi = f4(sdc / sdw, sdv / (sdw * sdw));
        ogi = f4(sgc / sgw, sgv / (sgw * sgw));
    }
    if (pair_out) st8(pair_out + 2 * i, odi, ogi);
    else { di_out[i] = odi; gi_out[i] = ogi; }
}

// ---------------------------------------------------------------------------------------------
// K22, tile-staged variant: the (TW+2·HL) x (TH+2·HL) pixel neighbourhood of a TW x TH output tile is
// brought into shared memory by three TMA tensor copies (surface_nd, DI colours, GI colours; one elected
// thread, one mbarrier), out-of-frame texels arrive as zeros (= the reference's `contains` test, because a
// zero depth skips the tap), and the 3x3 à-trous taps become LDS.128 at compile-time offsets.  HL = S + J,
// J = the largest |jitter| the blue-noise term can produce for stride S (0 for S <= 4, 1 for 8, 3 for 16).
// Same taps, same order, same arithmetic as k_denoise_wavelet: the two kernels are bit-identical in both
// arithmetic flavours (tests/test_gpu_parity.py::test_tiled_wavelet_matches_gather).
// ---------------------------------------------------------------------------------------------
ST_DEV u32 smem_addr(const void* p) { return (u32)__cvta_generic_to_shared(p); }
ST_DEV void mbar_init(u32 bar, u32 count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory"); }
ST_DEV void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
ST_DEV void mbar_expect_tx(u32 bar, u32 bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory"); }
ST_DEV bool mbar_try_wait(u32 bar, u32 parity) {
    u32 ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok != 0u;
}
ST_DEV void tma_load_2d(u32 dst, const CUtensorMap* tm, int c0, int c1, u32 bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 ::"r"(dst), "l"(reinterpret_cast<unsigned long long>(tm)), "r"(c0), "r"(c1), "r"(bar) : "memory");
}

// Per-centre state of K22: the terms of frame_denoising::sample_weight (frame_denoising.rs:363-392) that depend on the centre
// pixel only are evaluated once (1 / leeway of the depth ramp, sqrt of the centre luminances, the luminance sigmas); `geometry`
// is the part of a tap's weight shared by the DI and the GI signal, `add` the per-signal luminance term and the accumulation.
// Same expressions, same order as k_denoise_wavelet (both arithmetic flavours): bit-identical results.
template <bool FAST> struct WaveletCentre {
    float3 n; float depth, leeway, rcp_leeway, scdl, scgl, ls_di, ls_gi;
    float sdw; float3 sdc; float sdv; float sgw; float3 sgc; float sgv;
    ST_DEV void init(float4 cnd, float4 cdi, float4 cgi, float depth_sigma) {
        n = xyz(cnd); depth = cnd.w; leeway = cnd.w * depth_sigma; rcp_leeway = FAST ? sfu_rcp(leeway) : 0.0f;
        float3 cdc = xyz(cdi), cgc = xyz(cgi);
        scdl = sv_sqrt<FAST>(sv_luma<FAST>(cdc)); scgl = sv_sqrt<FAST>(sv_luma<FAST>(cgc));
        ls_di = lerpc(2.5f, 0.5f, sv_sqrt<FAST>(cdi.w)); ls_gi = lerpc(1.0f, 0.0f, sv_sqrt<FAST>(cgi.w));
        sdw = 1.0f; sdc = cdc; sdv = cdi.w; sgw = 1.0f; sgc = cgc; sgv = cgi.w;
    }
    // depth ramp and normal^64 of one tap (svgf_depth_weight / svgf_normal_weight); false = the tap cannot contribute
    ST_DEV bool geometry(float4 nds, float* dw, float* nw) const {
        float diff = fabs_(nds.w - depth);
        if (diff >= leeway) return false;
        *dw = FAST ? __fmaf_rn(-diff, rcp_leeway, 1.0f) : 1.0f - diff / leeway;
        *nw = svgf_normal_weight<FAST>(n, xyz(nds));
        return !(*dw == 0.0f || *nw == 0.0f);
    }
    ST_DEV void add(float dw, float nw, float4 sdi, float4 sgi) {
        if (FAST) {
            float dnw = dw * nw;
            float wd = svgf_luma_weight<true>(scdl, sv_luma<true>(xyz(sdi)), ls_di) * dnw;
            if (wd > 0.0f) { sdw += wd; sdc = f3(__fmaf_rn(wd, sdi.x, sdc.x), __fmaf_rn(wd, sdi.y, sdc.y), __fmaf_rn(wd, sdi.z, sdc.z)); sdv = __fmaf_rn(wd * wd, sdi.w, sdv); }
            float wg = svgf_luma_weight<true>(scgl, sv_luma<true>(xyz(sgi)), ls_gi) * dnw;
            if (wg > 0.0f) { sgw += wg; sgc = f3(__fmaf_rn(wg, sgi.x, sgc.x), __fmaf_rn(wg, sgi.y, sgc.y), __fmaf_rn(wg, sgi.z, sgc.z)); sgv = __fmaf_rn(wg * wg, sgi.w, sgv); }
        } else {
            float wd = svgf_luma_weight<false>(scdl, luma(xyz(sdi)), ls_di) * dw * nw;
            if (wd > 0.0f) { sdw += wd; sdc = sdc + wd * xyz(sdi); sdv += sq(wd) * sdi.w; }
            float wg = svgf_luma_weight<false>(scgl, luma(xyz(sgi)), ls_gi) * dw * nw;
            if (wg > 0.0f) { sgw += wg; sgc = sgc + wg * xyz(sgi); sgv += sq(wg) * sgi.w; }
        }
    }
    ST_DEV void store(float4* __restrict__ di_out, float4* __restrict__ gi_out, float4* __restrict__ pair_out, size_t i) const {
        float4 odi, ogi;
        if (FAST) {
            float rd = sfu_rcp(sdw), rg = sfu_rcp(sgw);
            odi = f4(sdc * rd, sdv * (rd * rd));
            ogi = f4(sgc * rg, sgv * (rg * rg));
        } else {
            odi = f4(sdc / sdw, sdv / (sdw * sdw));
            ogi = f4(sgc / sgw, sgv / (sgw * sgw));
        }
        if (pair_out) st8(pair_out + 2 * i, odi, ogi);   // interleaved {DI, GI} record for the wide-stride iterations (see k_denoise_wavelet)
        else { di_out[i] = odi; gi_out[i] = ogi; }
    }
};

template <int S, int J, int TW, int TH> struct WaveletTile {
    static constexpr int HL = S + J, BW = TW + 2 * HL, BH = TH + 2 * HL;
    static constexpr u32 BOX_BYTES = (u32)(BW * BH * 16);
    static constexpr u32 PLANE = (BOX_BYTES + 127u) & ~127u;
    static constexpr u32 SMEM = 3u * PLANE + 128u;   // + slack to align the first plane to 128 B
};

#ifndef ST_WAVELET_TILED_MINB
#define ST_WAVELET_TILED_MINB 1
#endif
template <bool FAST, int S, int J, int TW, int TH>
__global__ void __launch_bounds__(TW * TH, (TW * TH <= 256 && S <= 8) ? ST_WAVELET_TILED_MINB : 1) k_denoise_wavelet_tiled(KPARAMS, u32 frame, float strength,
                                                                   const __grid_constant__ CUtensorMap tm_nd, const __grid_constant__ CUtensorMap tm_di,
                                                                   const __grid_constant__ CUtensorMap tm_gi,
                                                                   float4* __restrict__ di_out, float4* __restrict__ gi_out, float4* __restrict__ pair_out,
                                                                   u32* __restrict__ errors) {
    typedef WaveletTile<S, J, TW, TH> T;
    extern __shared__ unsigned char s_raw[];
    __shared__ __align__(8) unsigned long long s_bar;
    const int tx = (int)threadIdx.x % TW, ty = (int)threadIdx.x / TW;
    const int x0 = (int)blockIdx.x * TW, y0 = cam.y0 + (int)blockIdx.y * TH;
    const u32 bar = smem_addr(&s_bar);
    const u32 raw = smem_addr(s_raw);
    const u32 base = (raw + 127u) & ~127u;
    if (threadIdx.x == 0) { mbar_init(bar, 1u); mbar_fence_init(); }
    __syncthreads();
    if (threadIdx.x == 0) {
        mbar_expect_tx(bar, 3u * T::BOX_BYTES);   // tensor coordinates: x in 8-byte elements (see wavelet_tensor_map), y in rows
        tma_load_2d(base, &tm_nd, (x0 - T::HL) * 2, y0 - T::HL, bar);
        tma_load_2d(base + T::PLANE, &tm_di, (x0 - T::HL) * 2, y0 - T::HL, bar);
        tma_load_2d(base + 2u * T::PLANE, &tm_gi, (x0 - T::HL) * 2, y0 - T::HL, bar);
    }
    const u32 px = (u32)(x0 + tx), py = (u32)(y0 + ty);
    const bool in = px < (u32)cam.w && py < (u32)cam.y1;
    int jo = 0;
    if (J > 0 && in) {   // the jitter only needs the blue-noise texel: fetched while the tile is in flight
        float4 bn = blue_noise(sc, px, py, frame);
        float2 jf = (f2(bn.z, bn.w) - f2(0.5f, 0.5f)) * ((float)S - 1.0f) * 0.5f;
        jo = to_i32_sat(jf.y) * T::BW + to_i32_sat(jf.x);
    }
    {   // every thread waits (the CTA's shared memory must stay allocated until the copies have landed)
        bool done = false;
        for (u32 spin = 0; spin < (1u << 20) && !done; spin++) done = mbar_try_wait(bar, 0u);
        if (!done) { if (threadIdx.x == 0) atomicAdd(errors, 1u); return; }
    }
    if (!in) return;
    const float4* __restrict__ t_nd = reinterpret_cast<const float4*>(s_raw + (base - raw));
    const float4* __restrict__ t_di = reinterpret_cast<const float4*>(s_raw + (base - raw) + T::PLANE);
    const float4* __restrict__ t_gi = reinterpret_cast<const float4*>(s_raw + (base - raw) + 2u * T::PLANE);
    const int c = (ty + T::HL) * T::BW + (tx + T::HL);
    const size_t i = pix(cam, px, py);
    float4 cnd = t_nd[c];
    float4 cdi = t_di[c];
    if (cnd.w == 0.0f) { if (pair_out) pair_out[2 * i] = f4(xyz(cdi), cdi.w); else di_out[i] = f4(xyz(cdi), cdi.w); return; }   // sky: DI passes through, GI is not written (frame_denoising.rs:248-254)
    WaveletCentre<FAST> ctr;
    ctr.init(cnd, cdi, t_gi[c], 0.33f / strength);   // depth sigma is the same for DI and GI (frame_denoising.rs:264,267)
    const int cj = c + jo;
#pragma unroll
    for (int oy = -1; oy <= 1; oy++) {
#pragma unroll
        for (int ox = -1; ox <= 1; ox++) {
            if (ox == 0 && oy == 0) continue;
            const int k = cj + oy * S * T::BW + ox * S;
            float4 nds = t_nd[k];
            if (nds.w == 0.0f) continue;   // sky, or outside the frame (zero-filled by the tensor copy)
            float dw, nw;
            if (!ctr.geometry(nds, &dw, &nw)) continue;
            ctr.add(dw, nw, t_di[k], t_gi[k]);
        }
    }
    ctr.store(di_out, gi_out, pair_out, i);
}

// R2 frame_composition::fs (frame_composition.rs:19-82) for pixel i: the linear HDR colour that k_composition stores and that
// k_taa_resolve composes into shared memory
ST_DEV float3 compose_px(const CameraDev& cam, const SceneDev& sc, int cur, u32 mode, const float4* __restrict__ di_diff, const float4* __restrict__ gi_diff, size_t i) {
    float3 color;
    if (mode == 0u) {
        GBuf g = gbuf_unpack(sc, cam.prim_gbuffer_d0[cur][i], cam.prim_gbuffer_d1[cur][i]);
        float3 dd = xyz(di_diff[i]), ds = xyz(cam.di_spec_samples[i]), gd = xyz(gi_diff[i]), gs = xyz(cam.gi_spec_samples[i]);
        if (g.depth != 0.0f) color = g.emissive + (dd + gd) * xyz(g.base_color) + ds + gs;
        else color = dd;
    } else if (mode == 1u) color = xyz(di_diff[i]);
    else if (mode == 2u) color = xyz(cam.di_spec_samples[i]);
    else if (mode == 3u) color = xyz(gi_diff[i]);
    else if (mode == 4u) color = xyz(cam.gi_spec_samples[i]);
    else if (mode == 5u) color = xyz(cam.ref_colors[i]);
    else if (mode == 6u) { float4 c = cam.ref_colors[i]; color = xyz(c) / c.w; }
    else color = f3s(0.f);
    return color;
}
// R2 frame_composition::fs (frame_composition.rs:19-82), linear HDR out
__global__ void __launch_bounds__(ST_BLOCK) k_composition(KPARAMS, int cur, u32 mode, const float4* __restrict__ di_diff, const float4* __restrict__ gi_diff) {
    Px p = pixel_full(cam);
    if (!p.in) return;
    size_t i = pix(cam, p.x, p.y);
    cam.output[i] = f4(compose_px(cam, sc, cur, mode, di_diff, gi_diff, i), 1.0f);
}

// ---- ST_OPT_TEMPORAL_AA (DESIGN.md §2 "Temporal anti-aliasing"): the resolve, in place of k_composition --------------------------
// Every step below is one IEEE operation in the order written (strict build only); oracle_taa/taa.cpp restates it operation for
// operation.  Colours are tonemapped, t(c) = c / (1 + max(c)), before they are boxed, filtered and blended.
#define TAA_TW 32
#define TAA_TH 8
static const float kTaaClipEps = 1e-8f;   // added to the box's half extent (Playdead's clip_aabb)
ST_DEV float taa_max(float a, float b) { return a > b ? a : b; }
ST_DEV float taa_min(float a, float b) { return a < b ? a : b; }
ST_DEV float3 taa_tonemap(float3 c) { const float d = 1.0f + taa_max(taa_max(c.x, c.y), c.z); return f3(c.x / d, c.y / d, c.z / d); }
ST_DEV float3 taa_untonemap(float3 t) { const float d = 1.0f - taa_max(taa_max(t.x, t.y), t.z); return f3(t.x / d, t.y / d, t.z / d); }
ST_DEV float3 taa_ycocg(float3 c) { return f3((0.25f * c.x + 0.5f * c.y) + 0.25f * c.z, 0.5f * c.x - 0.5f * c.z, (-0.25f * c.x + 0.5f * c.y) - 0.25f * c.z); }
ST_DEV float3 taa_rgb(float3 v) { const float t = v.x - v.z; return f3(t + v.y, v.x + v.z, t - v.y); }
// Catmull-Rom weights of the four taps around a sample at fraction f past the second one
ST_DEV void taa_cr_weights(float f, float w[4]) {
    w[0] = f * (-0.5f + f * (1.0f - 0.5f * f));
    w[1] = 1.0f + (f * f) * (-2.5f + 1.5f * f);
    w[2] = f * (0.5f + f * (2.0f - 1.5f * f));
    w[3] = (f * f) * (-0.5f + 0.5f * f);
}
// `jit` = (J(f), J(f - 1)) in pixels; cam.curr / cam.prev are the jittered cameras of this frame and the last
__global__ void __launch_bounds__(TAA_TW * TAA_TH) k_taa_resolve(KPARAMS, int cur, u32 mode, const float4* __restrict__ di_diff, const float4* __restrict__ gi_diff,
                                                                 const float4* __restrict__ hist_in, float4* __restrict__ hist_out, float4 jit) {
    const int HW = TAA_TW + 2, HH = TAA_TH + 2;
    __shared__ float4 s_t[HW * HH];   // tonemapped composed colours of the tile and a 1-pixel halo, taps clamped to the screen
    const int bx = (int)blockIdx.x * TAA_TW - 1, by = (int)blockIdx.y * TAA_TH - 1;
    for (int k = threadIdx.x; k < HW * HH; k += TAA_TW * TAA_TH) {
        const int x = min(max(bx + k % HW, 0), cam.w - 1), y = min(max(by + k / HW, 0), cam.h - 1);
        s_t[k] = f4(taa_tonemap(compose_px(cam, sc, cur, mode, di_diff, gi_diff, pix(cam, (u32)x, (u32)y))), 0.0f);
    }
    __syncthreads();
    const int tx = threadIdx.x % TAA_TW, ty = threadIdx.x / TAA_TW;
    const u32 px = blockIdx.x * TAA_TW + tx, py = blockIdx.y * TAA_TH + ty;
    if (px >= (u32)cam.w || py >= (u32)cam.h) return;
    const size_t i = pix(cam, px, py);
    // 1-2. the current value and the 3x3 box in YCoCg (row by row)
    const float3 t = xyz(s_t[(ty + 1) * HW + tx + 1]);
    float3 lo = taa_ycocg(xyz(s_t[ty * HW + tx])), hi = lo;
#pragma unroll
    for (int k = 1; k < 9; k++) {
        const float3 v = taa_ycocg(xyz(s_t[(ty + k / 3) * HW + tx + k % 3]));
        lo = f3(taa_min(lo.x, v.x), taa_min(lo.y, v.y), taa_min(lo.z, v.z)); hi = f3(taa_max(hi.x, v.x), taa_max(hi.y, v.y), taa_max(hi.z, v.z));
    }
    // 3. where the surface seen through the unjittered pixel centre was in last frame's unjittered screen
    const float W = cam.curr.screen.x, H = cam.curr.screen.y;
    float2 q; bool ok = true;
    if (cam.prim_gbuffer_d0[cur][i].x != 0.0f) {
        const float4 v = cam.velocity_map[i];
        q = f2((((float)px + 0.5f) - v.x) - (jit.x - jit.z), (((float)py + 0.5f) - v.y) - (jit.y - jit.w));
    } else {   // sky: the direction through the unjittered centre (jittered screen point p + 0.5 - J(f)), at w = 0 through last frame's camera
        const float sx = ((float)px + 0.5f) - jit.x, sy = ((float)py + 0.5f) - jit.y;
        const float nx = sx * 2.0f / W - 1.0f, ny = -(sy * 2.0f / H - 1.0f);
        const float3 far_plane = project_point(cam_n2w(cam.curr), f3(nx, ny, kF32Eps)), near_plane = project_point(cam_n2w(cam.curr), f3(nx, ny, 1.0f));
        const float4 clip = mat_mul(cam_pv(cam.prev), f4(norm(far_plane - near_plane), 0.0f));
        const float2 s = cam_clip_to_screen(cam.prev, clip);
        q = f2(s.x + jit.z, s.y + jit.w);
        ok = clip.w > 0.0f;
    }
    // 4. validity: on screen, and a non-zero count at the nearest history texel
    ok = ok && q.x >= 0.0f && q.y >= 0.0f && q.x < W && q.y < H;
    float n = 0.0f;
    if (ok) n = hist_in[pix(cam, (u32)floorf(q.x), (u32)floorf(q.y))].w;
    float3 h = t;
    if (n > 0.0f) {
        // 5. separable 4x4 Catmull-Rom over the tonemapped history, texel centres at i + 0.5, taps clamped to the screen
        const float ux = q.x - 0.5f, uy = q.y - 0.5f, fx0 = floorf(ux), fy0 = floorf(uy);
        float wx[4], wy[4];
        taa_cr_weights(ux - fx0, wx); taa_cr_weights(uy - fy0, wy);
        const int ix = (int)fx0 - 1, iy = (int)fy0 - 1;
        h = f3s(0.0f);
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const u32 yy = (u32)min(max(iy + j, 0), cam.h - 1);
            float3 row = f3s(0.0f);
#pragma unroll
            for (int k = 0; k < 4; k++) row = row + wx[k] * xyz(hist_in[pix(cam, (u32)min(max(ix + k, 0), cam.w - 1), yy)]);
            h = h + wy[j] * row;
        }
        // 6. clip toward the box centre, into the box (YCoCg)
        const float3 c = 0.5f * (hi + lo), e = 0.5f * (hi - lo) + f3s(kTaaClipEps);
        const float3 d = taa_ycocg(h) - c;
        const float m = taa_max(taa_max(fabs_(d.x / e.x), fabs_(d.y / e.y)), fabs_(d.z / e.z));
        if (m > 1.0f) h = taa_rgb(c + d / m);
    } else n = 0.0f;
    // 7-8. blend, count, store
    const float a = 1.0f / (n + 1.0f), alpha = a > 0.1f ? a : 0.1f;
    const float3 r = (1.0f - alpha) * h + alpha * t;
    const float n1 = n + 1.0f;
    hist_out[i] = f4(r, n1 < 16.0f ? n1 : 16.0f);
    cam.output[i] = f4(taa_untonemap(r), 1.0f);
}


// Rgba8UnormSrgb store of the composed frame (the reference's default CameraViewport::format,
// strolle/src/camera.rs:177-185): clamp to [0,1], sRGB OETF, round to nearest.
__global__ void __launch_bounds__(ST_BLOCK) k_output_rgba8(KPARAMS, uchar4* __restrict__ out) {
    Px p = pixel_full(cam);
    if (!p.in) return;
    size_t i = pix(cam, p.x, p.y);
    float4 c = cam.output[i];
    float v[3] = {c.x, c.y, c.z};
    u32 q[3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        float x = sat(v[k]);
        float e = (x <= 0.0031308f) ? 12.92f * x : 1.055f * pow_det(x, 1.0f / 2.4f) - 0.055f;
        q[k] = to_u32_sat(sat(e) * 255.0f + 0.5f);
    }
    out[i] = make_uchar4((unsigned char)q[0], (unsigned char)q[1], (unsigned char)q[2], 255);
}

// ---- ST_OPT_TONEMAPPING / ST_OPT_AUTO_EXPOSURE (DESIGN.md §2 "Exposure and tonemapping") --------------------------------------------
// Every f32 step is one IEEE operation in the order written (strict build only); oracle_exposure/exposure.cpp restates it operation for
// operation.  The metering's doubles use + - * / floor ceil only, which are correctly rounded on the host and the device alike.
// The histogram's shape (DESIGN.md §4 "Exposure and tonemapping" compares the variants; tools/exposure_variants.py builds them): threads
// per CTA, CTAs per SM, lanes merged per bin with __match_any_sync (1) or a shared atomicAdd per lane (0), the metering in the last CTA
// (0) or in a second one-CTA launch (1).  The defaults are the fastest measured.
#ifndef ST_EXPO_THREADS
#define ST_EXPO_THREADS 512
#endif
#ifndef ST_EXPO_CTAS_PER_SM
#define ST_EXPO_CTAS_PER_SM 4
#endif
#ifndef ST_EXPO_AGGREGATE
#define ST_EXPO_AGGREGATE 1
#endif
#ifndef ST_EXPO_METER_LAUNCH
#define ST_EXPO_METER_LAUNCH 0
#endif
#define EXPO_THREADS ST_EXPO_THREADS
#define EXPO_WARPS (EXPO_THREADS / 32)
ST_DEV float expo_luminance(float r, float g, float b) { return (0.2126f * r + 0.7152f * g) + 0.0722f * b; }
// The histogram bin of luminance L (256 bins of 1/8 stop over log2 L in [-16, 16)), or -1 where the pixel does not count
ST_DEV int expo_bin(float L) {
    if (!(L > 0.0f) || L == finf()) return -1;
    const float y = (log2_x(L) + 16.0f) * 8.0f;
    return y < 0.0f ? 0 : (y >= 256.0f ? 255 : (int)y);
}
// The metering and adaptation of DESIGN.md §2, by one thread over the frame's 256 bin counts
ST_DEV void expo_meter(const u32* bins, u32* state, const ExposureDev& p) {
    unsigned long long n = 0;
    for (int b = 0; b < kExposureBins; b++) n += bins[b];
    const double lo = floor((double)p.low * (double)n), hi = ceil((double)p.high * (double)n);
    double start = 0.0, kept = 0.0, sum = 0.0;
    for (int b = 0; b < kExposureBins; b++) {
        const double end = start + (double)bins[b];
        const double a = start > lo ? start : lo, z = end < hi ? end : hi;
        if (z > a) { kept = kept + (z - a); sum = sum + (z - a) * (-16.0 + ((double)b + 0.5) / 8.0); }
        start = end;
    }
    const bool first = state[4] == 0u;
    const float prev = __uint_as_float(state[0]);
    float target;
    if (kept > 0.0) {
        double t = sum / kept - (-2.4739311883324122);   // - log2(0.18): an average of mid-grey meters EV 0
        t = t < (double)p.ev_min ? (double)p.ev_min : t;
        t = t > (double)p.ev_max ? (double)p.ev_max : t;
        target = (float)t;
    } else if (first) target = rclamp(0.0f, p.ev_min, p.ev_max);
    else target = prev;
    float ev = target;
    if (!first) {
        const float d = target - prev;
        if (d > p.speed_up) ev = prev + p.speed_up;
        else if (d < -p.speed_down) ev = prev - p.speed_down;
    }
    state[0] = __float_as_uint(ev); state[1] = __float_as_uint(target);
    state[2] = (u32)n; state[3] = (u32)kept; state[4] = state[4] + 1u;
}
// One thread per pixel over grid-stride rounds.  Lanes of a warp that fall into one bin (a sky, a flat wall) are merged by
// __match_any_sync and counted once, by their lowest lane, into the warp's own shared sub-histogram; each CTA then adds its non-zero
// bins to the accumulator with one global atomic each.  The last CTA to finish (ticket after a fence) meters.
__global__ void __launch_bounds__(EXPO_THREADS) k_exposure_histogram(const float4* __restrict__ output, u32 n, u32* __restrict__ state, ExposureDev p) {
    __shared__ u32 s_hist[EXPO_WARPS][kExposureBins];
    __shared__ bool s_last;
    const u32 lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    for (u32 k = threadIdx.x; k < EXPO_WARPS * kExposureBins; k += EXPO_THREADS) (&s_hist[0][0])[k] = 0u;
    __syncthreads();
    for (u32 base = blockIdx.x * EXPO_THREADS; base < n; base += gridDim.x * EXPO_THREADS) {   // base is uniform: whole warps take part
        const u32 i = base + threadIdx.x;
        int bin = -1;
        if (i < n) { const float4 c = output[i]; bin = expo_bin(expo_luminance(c.x, c.y, c.z)); }
#if ST_EXPO_AGGREGATE
        const u32 same = __match_any_sync(0xffffffffu, bin);
        if (bin >= 0 && lane == (u32)(__ffs(same) - 1)) s_hist[warp][bin] += (u32)__popc(same);   // the warp's own row: no other writer
        __syncwarp();
#else
        if (bin >= 0) atomicAdd(&s_hist[warp][bin], 1u);
        (void)lane;
#endif
    }
    __syncthreads();
    for (u32 b = threadIdx.x; b < kExposureBins; b += EXPO_THREADS) {
        u32 c = 0;
#pragma unroll
        for (int w = 0; w < EXPO_WARPS; w++) c += s_hist[w][b];
        if (c) atomicAdd(&state[kExposureAccum + b], c);
    }
#if ST_EXPO_METER_LAUNCH
    (void)s_last; (void)p;
#else
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_last = atomicAdd(&state[kExposureTicket], 1u) == gridDim.x - 1u;
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    u32* bins = &s_hist[0][0];   // the frame's counts; the accumulator is left zero for the next frame
    for (u32 b = threadIdx.x; b < kExposureBins; b += EXPO_THREADS) { bins[b] = atomicExch(&state[kExposureAccum + b], 0u); state[5 + b] = bins[b]; }
    __syncthreads();
    if (threadIdx.x == 0) { expo_meter(bins, state, p); state[kExposureTicket] = 0u; }
#endif
}
#if ST_EXPO_METER_LAUNCH
__global__ void __launch_bounds__(kExposureBins) k_exposure_meter(u32* __restrict__ state, ExposureDev p) {
    __shared__ u32 bins[kExposureBins];
    bins[threadIdx.x] = state[kExposureAccum + threadIdx.x];
    state[kExposureAccum + threadIdx.x] = 0u; state[5 + threadIdx.x] = bins[threadIdx.x];
    __syncthreads();
    if (threadIdx.x == 0) expo_meter(bins, state, p);
}
#endif

// The display transforms T of ST_OPT_TONEMAPPING 2..4 (1 is the identity)
ST_DEV float3 expo_mat(const float m[9], float3 v) {
    return f3((m[0] * v.x + m[1] * v.y) + m[2] * v.z, (m[3] * v.x + m[4] * v.y) + m[5] * v.z, (m[6] * v.x + m[7] * v.y) + m[8] * v.z);
}
ST_DEV float expo_aces_rrt_odt(float v) { return (v * (v + 0.0245786f) - 0.000090537f) / (v * (0.983729f * v + 0.4329510f) + 0.238081f); }
ST_DEV float expo_agx_curve(float v) {
    float l = v > 0.0f ? log2_x(v) : -12.47393f;
    l = l < -12.47393f ? -12.47393f : l;
    l = l > 4.026069f ? 4.026069f : l;
    const float x = (l + 12.47393f) / 16.499999f;
    const float x2 = x * x, x4 = x2 * x2;
    return (((((15.5f * x4 * x2 - 40.14f * x4 * x) + 31.96f * x4) - 6.868f * x2 * x) + 0.4298f * x2) + 0.1191f * x) - 0.00232f;
}
template <int OP>
ST_DEV float3 expo_transform(float3 x) {
    if (OP == 2) { const float d = 1.0f + expo_luminance(x.x, x.y, x.z); return f3(x.x / d, x.y / d, x.z / d); }
    if (OP == 3) {
        const float A[9] = {0.59719f, 0.35458f, 0.04823f, 0.07600f, 0.90834f, 0.01566f, 0.02840f, 0.13383f, 0.83777f};
        const float B[9] = {1.60475f, -0.53108f, -0.07367f, -0.10208f, 1.10813f, -0.00605f, -0.00327f, -0.07276f, 1.07602f};
        const float3 v = expo_mat(A, x);
        return expo_mat(B, f3(expo_aces_rrt_odt(v.x), expo_aces_rrt_odt(v.y), expo_aces_rrt_odt(v.z)));
    }
    if (OP == 4) {
        const float M[9] = {0.842479062253094f, 0.0784335999999992f, 0.0792237451477643f, 0.0423282422610123f, 0.878468636469772f, 0.0791661274605434f,
                            0.0423756549057051f, 0.0784336f, 0.879142973793104f};
        const float MI[9] = {1.19687900512017f, -0.0980208811401368f, -0.0990297440797205f, -0.0528968517574562f, 1.15190312990417f, -0.0989611768448433f,
                             -0.0529716355144438f, -0.0980434501171241f, 1.15107367264116f};
        const float3 v = expo_mat(M, x);
        const float3 u = expo_mat(MI, f3(expo_agx_curve(v.x), expo_agx_curve(v.y), expo_agx_curve(v.z)));
        return f3(pow_det(u.x > 0.0f ? u.x : 0.0f, 2.2f), pow_det(u.y > 0.0f ? u.y : 0.0f, 2.2f), pow_det(u.z > 0.0f ? u.z : 0.0f, 2.2f));
    }
    return x;
}
// The Rgba8UnormSrgb store of k_output_rgba8 after exposure and T
template <int OP>
__global__ void __launch_bounds__(ST_BLOCK) k_output_display(KPARAMS, uchar4* __restrict__ out, const u32* __restrict__ state, ExposureDev ep) {
    Px p = pixel_full(cam);
    if (!p.in) return;
    size_t i = pix(cam, p.x, p.y);
    const float ev = state ? __uint_as_float(state[0]) : ep.ev;
    const float s = pow_det(2.0f, ep.compensation - ev);
    const float4 c = cam.output[i];
    const float3 t = expo_transform<OP>(f3((c.x > 0.0f ? c.x : 0.0f) * s, (c.y > 0.0f ? c.y : 0.0f) * s, (c.z > 0.0f ? c.z : 0.0f) * s));
    float v[3] = {t.x, t.y, t.z};
    u32 q[3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        float x = sat(v[k]);
        float e = (x <= 0.0031308f) ? 12.92f * x : 1.055f * pow_det(x, 1.0f / 2.4f) - 0.055f;
        q[k] = to_u32_sat(sat(e) * 255.0f + 0.5f);
    }
    out[i] = make_uchar4((unsigned char)q[0], (unsigned char)q[1], (unsigned char)q[2], 255);
}

// ---- ST_OPT_BLOOM (DESIGN.md §2 "Bloom") -------------------------------------------------------------------------------------------
// Every f32 step is one IEEE operation in the order written (strict build only); oracle_bloom/bloom.cpp restates it operation for
// operation.  The small levels' shape (DESIGN.md §4 "Bloom" compares the variants; tools/bloom_variants.py builds them): one launch per
// level, down and up (ST_BLOOM_TAIL_TEXELS 0), or the levels of at most ST_BLOOM_TAIL_TEXELS texels down and back up in one launch:
// ST_BLOOM_TAIL_KIND 0, one CTA over global memory; 1, one CTA holding the tail in its shared memory; 2, a cluster of
// ST_BLOOM_CLUSTER CTAs holding it in distributed shared memory.  Every shape computes each texel with the same functions; one launch
// per level measured fastest.
#ifndef ST_BLOOM_TAIL_TEXELS
#define ST_BLOOM_TAIL_TEXELS 0
#endif
#ifndef ST_BLOOM_TAIL_KIND
#define ST_BLOOM_TAIL_KIND 0
#endif
#ifndef ST_BLOOM_CLUSTER
#define ST_BLOOM_CLUSTER 8
#endif
#define BLOOM_TX 32   // level-0 texels per CTA (x, y) of the first downsample
#define BLOOM_TY 8
#define BLOOM_SX (2 * BLOOM_TX + 4)   // the frame texels it reads: its 2 x 2 footprints plus a 2-texel halo
#define BLOOM_SY (2 * BLOOM_TY + 4)
#define BLOOM_TAIL_THREADS 512
ST_DEV int bloom_clampi(int v, int hi) { return v < 0 ? 0 : (v > hi ? hi : v); }
// One channel of the frame: c where it is finite and > 0, else 0; times the exposure
ST_DEV float bloom_in(float c, float s) { return (c > 0.0f && c < finf()) ? c * s : 0.0f; }
// A frame texel as the pyramid takes it: cleared, exposed, through the soft-knee prefilter (threshold > 0); a non-finite channel is 0
ST_DEV float4 bloom_input(float4 c, float s, const BloomDev& b) {
    float x = bloom_in(c.x, s), y = bloom_in(c.y, s), z = bloom_in(c.z, s);
    if (b.threshold > 0.0f) {
        float m = x > y ? x : y;
        m = m > z ? m : z;
        const float t = b.threshold, k = t * b.softness;
        const float q0 = rclamp((m - t) + k, 0.0f, 2.0f * k);
        const float q = (q0 * q0) / (4.0f * k + 1e-4f);
        const float w = (q > m - t ? q : m - t) / (m > 1e-4f ? m : 1e-4f);
        x = x * w; y = y * w; z = z * w;
    }
    return f4(x < finf() ? x : 0.0f, y < finf() ? y : 0.0f, z < finf() ? z : 0.0f, 0.0f);
}
// The 2 x 2 box of one of the 13 taps, as {w t, w} with t its average and w its Karis weight 1 / (1 + L(t)) (KARIS) or 1
template <bool KARIS>
ST_DEV float4 bloom_tap(float4 a, float4 b, float4 c, float4 d) {
    const float4 t = ((a + b) + (c + d)) * 0.25f;
    if (!KARIS) return f4(t.x, t.y, t.z, 1.0f);
    const float w = 1.0f / (1.0f + expo_luminance(t.x, t.y, t.z));
    return f4(t.x * w, t.y * w, t.z * w, w);
}
// A group of four taps (row-major): their weighted average
template <bool KARIS>
ST_DEV float4 bloom_group(float4 a, float4 b, float4 c, float4 d) {
    const float4 s = (a + b) + (c + d);
    if (!KARIS) return f4(s.x * 0.25f, s.y * 0.25f, s.z * 0.25f, 0.0f);
    const float w = (a.w + b.w) + (c.w + d.w);
    return f4(s.x / w, s.y / w, s.z / w, 0.0f);
}
// The 13-tap texel from odd-corner taps o[n][m] (corners 2i - 1 + 2m, 2j - 1 + 2n) and even-corner taps e[n][m] (2i + 2m, 2j + 2n)
template <bool KARIS, class O, class E>
ST_DEV float4 bloom_13(O o, E e) {
    const float4 C = bloom_group<KARIS>(e(0, 0), e(1, 0), e(0, 1), e(1, 1));
    const float4 TL = bloom_group<KARIS>(o(0, 0), o(1, 0), o(0, 1), o(1, 1)), TR = bloom_group<KARIS>(o(1, 0), o(2, 0), o(1, 1), o(2, 1));
    const float4 BL = bloom_group<KARIS>(o(0, 1), o(1, 1), o(0, 2), o(1, 2)), BR = bloom_group<KARIS>(o(1, 1), o(2, 1), o(1, 2), o(2, 2));
    const float4 r = C * 0.5f + ((TL + TR) + (BL + BR)) * 0.125f;
    return f4(r.x, r.y, r.z, 0.0f);
}
// Level k >= 1: texel (i, j) from level k - 1 (sw x sh, texel t read as src(t)), every index clamped
template <class S>
ST_DEV float4 bloom_down_at(S src, int sw, int sh, int i, int j) {
    auto T = [&](int x, int y) { return src((size_t)bloom_clampi(y, sh - 1) * sw + bloom_clampi(x, sw - 1)); };
    auto tap = [&](int cx, int cy) { return bloom_tap<false>(T(cx - 1, cy - 1), T(cx, cy - 1), T(cx - 1, cy), T(cx, cy)); };
    return bloom_13<false>([&](int m, int n) { return tap(2 * i - 1 + 2 * m, 2 * j - 1 + 2 * n); },
                           [&](int m, int n) { return tap(2 * i + 2 * m, 2 * j + 2 * n); });
}
// Plain loads: the tails read what their own CTA wrote
ST_DEV float4 bloom_down_texel(const float4* src, int sw, int sh, int i, int j) { return bloom_down_at([&](size_t t) { return src[t]; }, sw, sh, i, j); }
// tent(u)(fx, fy): the 3 x 3 (1 2 1) x (1 2 1) / 16 filter of the coarse level u (cw x ch) at the texel (min(fx >> 1, cw - 1),
// min(fy >> 1, ch - 1)) that covers the fine texel, every index clamped
template <class S>
ST_DEV float4 bloom_tent_at(S u, int cw, int ch, int fx, int fy) {
    const int cx = (fx >> 1) < cw - 1 ? (fx >> 1) : cw - 1, cy = (fy >> 1) < ch - 1 ? (fy >> 1) : ch - 1;
    const int x0 = bloom_clampi(cx - 1, cw - 1), x2 = bloom_clampi(cx + 1, cw - 1);
    float4 r[3];
#pragma unroll
    for (int d = 0; d < 3; d++) {
        const size_t row = (size_t)bloom_clampi(cy - 1 + d, ch - 1) * cw;
        r[d] = (u(row + x0) + u(row + cx) * 2.0f) + u(row + x2);
    }
    return ((r[0] + r[1] * 2.0f) + r[2]) * 0.0625f;
}
ST_DEV float4 bloom_tent(const float4* u, int cw, int ch, int fx, int fy) { return bloom_tent_at([&](size_t t) { return u[t]; }, cw, ch, fx, fy); }
// up_k(i, j) = (1 - a) down_k + a tent(up_{k+1})
template <class D, class C>
ST_DEV float4 bloom_up_at(D down, C coarse, int w, int cw, int ch, int i, int j, float a) {
    const float4 t = bloom_tent_at(coarse, cw, ch, i, j);
    const float4 r = down((size_t)j * w + i) * (1.0f - a) + t * a;
    return f4(r.x, r.y, r.z, 0.0f);
}
ST_DEV float4 bloom_up_texel(const float4* down, const float4* coarse, int w, int cw, int ch, int i, int j, float a) {
    return bloom_up_at([&](size_t t) { return down[t]; }, [&](size_t t) { return coarse[t]; }, w, cw, ch, i, j, a);
}
// The first downsample, frame -> level 0 (dw x dh), BLOOM_TX x BLOOM_TY texels per CTA.  The CTA's frame texels (footprints plus the
// 2-texel halo) are loaded once, through the input rule, into shared memory; then the 13 taps' boxes, each once with its Karis weight;
// then each texel's groups.
__global__ void __launch_bounds__(BLOOM_TX * BLOOM_TY) k_bloom_down0(const float4* __restrict__ output, int W, int H, float4* __restrict__ dst, int dw, int dh,
                                                                     const u32* __restrict__ state, ExposureDev ep, int tm, BloomDev bp) {
    __shared__ float4 s_src[BLOOM_SY][BLOOM_SX];
    __shared__ float4 s_odd[BLOOM_TY + 2][BLOOM_TX + 2];    // corner (2 i0 - 1 + 2 m, 2 j0 - 1 + 2 n)
    __shared__ float4 s_even[BLOOM_TY + 1][BLOOM_TX + 1];   // corner (2 i0 + 2 m, 2 j0 + 2 n)
    const int i0 = blockIdx.x * BLOOM_TX, j0 = blockIdx.y * BLOOM_TY, x0 = 2 * i0 - 2, y0 = 2 * j0 - 2;
    float s = 1.0f;
    if (tm != 0) s = pow_det(2.0f, ep.compensation - (state ? __uint_as_float(state[0]) : ep.ev));
    for (int k = threadIdx.x; k < BLOOM_SY * BLOOM_SX; k += BLOOM_TX * BLOOM_TY) {
        const int ly = k / BLOOM_SX, lx = k - ly * BLOOM_SX;
        (&s_src[0][0])[k] = bloom_input(output[(size_t)bloom_clampi(y0 + ly, H - 1) * W + bloom_clampi(x0 + lx, W - 1)], s, bp);
    }
    __syncthreads();
    for (int k = threadIdx.x; k < (BLOOM_TY + 2) * (BLOOM_TX + 2); k += BLOOM_TX * BLOOM_TY) {
        const int n = k / (BLOOM_TX + 2), m = k - n * (BLOOM_TX + 2);
        s_odd[n][m] = bloom_tap<true>(s_src[2 * n][2 * m], s_src[2 * n][2 * m + 1], s_src[2 * n + 1][2 * m], s_src[2 * n + 1][2 * m + 1]);
    }
    for (int k = threadIdx.x; k < (BLOOM_TY + 1) * (BLOOM_TX + 1); k += BLOOM_TX * BLOOM_TY) {
        const int n = k / (BLOOM_TX + 1), m = k - n * (BLOOM_TX + 1);
        s_even[n][m] = bloom_tap<true>(s_src[2 * n + 1][2 * m + 1], s_src[2 * n + 1][2 * m + 2], s_src[2 * n + 2][2 * m + 1], s_src[2 * n + 2][2 * m + 2]);
    }
    __syncthreads();
    const int li = threadIdx.x % BLOOM_TX, lj = threadIdx.x / BLOOM_TX, i = i0 + li, j = j0 + lj;
    if (i >= dw || j >= dh) return;
    dst[(size_t)j * dw + i] = bloom_13<true>([&](int m, int n) { return s_odd[lj + n][li + m]; }, [&](int m, int n) { return s_even[lj + n][li + m]; });
}
__global__ void __launch_bounds__(ST_BLOCK) k_bloom_down(const float4* __restrict__ src, int sw, int sh, float4* __restrict__ dst, int dw, int dh) {
    const int i = blockIdx.x * TILE_W + threadIdx.x % TILE_W, j = blockIdx.y * TILE_H + threadIdx.x / TILE_W;
    if (i < dw && j < dh) dst[(size_t)j * dw + i] = bloom_down_texel(src, sw, sh, i, j);
}
__global__ void __launch_bounds__(ST_BLOCK) k_bloom_up(const float4* __restrict__ down, const float4* __restrict__ coarse, int w, int h, int cw, int ch,
                                                       float4* __restrict__ up, float a) {
    const int i = blockIdx.x * TILE_W + threadIdx.x % TILE_W, j = blockIdx.y * TILE_H + threadIdx.x / TILE_W;
    if (i < w && j < h) up[(size_t)j * w + i] = bloom_up_texel(down, coarse, w, cw, ch, i, j, a);
}
// Levels first .. L - 1 down from level first - 1, then up_{L-2} .. up_first, by one CTA: each level is one block-wide pass over
// global memory (L1 / L2 resident at these sizes), separated by __syncthreads
__global__ void __launch_bounds__(BLOOM_TAIL_THREADS) k_bloom_tail(const __grid_constant__ BloomLevels lv, int first, float a) {
    for (int k = first; k < lv.levels; k++) {
        for (int t = threadIdx.x; t < lv.w[k] * lv.h[k]; t += BLOOM_TAIL_THREADS) {
            const int j = t / lv.w[k], i = t - j * lv.w[k];
            lv.down[k][t] = bloom_down_texel(lv.down[k - 1], lv.w[k - 1], lv.h[k - 1], i, j);
        }
        __syncthreads();
    }
    for (int k = lv.levels - 2; k >= first; k--) {
        for (int t = threadIdx.x; t < lv.w[k] * lv.h[k]; t += BLOOM_TAIL_THREADS) {
            const int j = t / lv.w[k], i = t - j * lv.w[k];
            lv.up[k][t] = bloom_up_texel(lv.down[k], lv.up[k + 1], lv.w[k], lv.w[k + 1], lv.h[k + 1], i, j, a);
        }
        __syncthreads();
    }
}
#if ST_BLOOM_TAIL_KIND == 1
// The same tail held in the CTA's dynamic shared memory: down_first .. down_{L-1}, then up_first .. up_{L-2}; only level first - 1 is
// read from global memory, every level is also written there (the "bloom" read-back)
__global__ void __launch_bounds__(BLOOM_TAIL_THREADS) k_bloom_tail_smem(const __grid_constant__ BloomLevels lv, int first, float a) {
    extern __shared__ float4 s_lv[];
    const int L = lv.levels;
    auto base = [&](bool up, int k) {   // offset of a level in s_lv
        size_t off = 0;
        for (int q = first; q < L; q++) { if (!up && q == k) return off; off += (size_t)lv.w[q] * lv.h[q]; }
        for (int q = first; q + 1 < L; q++) { if (q == k) return off; off += (size_t)lv.w[q] * lv.h[q]; }
        return off;
    };
    for (int k = first; k < L; k++) {
        const float4* sp = s_lv + base(false, k - 1);
        float4* d = s_lv + base(false, k);
        for (int t = threadIdx.x; t < lv.w[k] * lv.h[k]; t += BLOOM_TAIL_THREADS) {
            const int j = t / lv.w[k], i = t - j * lv.w[k];
            const float4 v = k == first ? bloom_down_texel(lv.down[k - 1], lv.w[k - 1], lv.h[k - 1], i, j) : bloom_down_texel(sp, lv.w[k - 1], lv.h[k - 1], i, j);
            d[t] = v; lv.down[k][t] = v;
        }
        __syncthreads();
    }
    for (int k = L - 2; k >= first; k--) {
        const float4* sd = s_lv + base(false, k);
        const float4* sc = s_lv + (k + 1 == L - 1 ? base(false, k + 1) : base(true, k + 1));
        float4* u = s_lv + base(true, k);
        for (int t = threadIdx.x; t < lv.w[k] * lv.h[k]; t += BLOOM_TAIL_THREADS) {
            const int j = t / lv.w[k], i = t - j * lv.w[k];
            const float4 v = bloom_up_texel(sd, sc, lv.w[k], lv.w[k + 1], lv.h[k + 1], i, j, a);
            u[t] = v; lv.up[k][t] = v;
        }
        __syncthreads();
    }
}
#endif
#if ST_BLOOM_TAIL_KIND == 2
// The same tail spread over a cluster of ST_BLOOM_CLUSTER CTAs: texel t of a level of n texels lives in the shared memory of rank
// t / ceil(n / ST_BLOOM_CLUSTER); each rank computes its own texels, reads the others' through distributed shared memory, and the cluster
// synchronises between levels.  Only level first - 1 is read from global memory; every level is also written there.
__global__ void __launch_bounds__(BLOOM_TAIL_THREADS) k_bloom_tail_cluster(const __grid_constant__ BloomLevels lv, int first, float a) {
    namespace cg = cooperative_groups;
    cg::cluster_group cluster = cg::this_cluster();
    extern __shared__ float4 s_lv[];
    const int L = lv.levels, R = (int)cluster.block_rank();
    auto chunk = [&](int k) { return (lv.w[k] * lv.h[k] + ST_BLOOM_CLUSTER - 1) / ST_BLOOM_CLUSTER; };
    auto base = [&](bool up, int k) {   // offset of a level's chunk in s_lv (the same in every rank)
        size_t off = 0;
        for (int q = first; q < L; q++) { if (!up && q == k) return off; off += (size_t)chunk(q); }
        for (int q = first; q + 1 < L; q++) { if (q == k) return off; off += (size_t)chunk(q); }
        return off;
    };
    auto dsm = [&](size_t b, int c) {   // texel t of the level whose chunks start at b
        return [&cluster, b, c](size_t t) { const unsigned r = (unsigned)(t / (size_t)c); return *cluster.map_shared_rank(s_lv + b + (t - (size_t)r * c), r); };
    };
    for (int k = first; k < L; k++) {
        const int c = chunk(k), n = lv.w[k] * lv.h[k];
        float4* d = s_lv + base(false, k);
        for (int t = R * c + threadIdx.x; t < min(n, (R + 1) * c); t += BLOOM_TAIL_THREADS) {
            const int j = t / lv.w[k], i = t - j * lv.w[k];
            const float4 v = k == first ? bloom_down_texel(lv.down[k - 1], lv.w[k - 1], lv.h[k - 1], i, j)
                                        : bloom_down_at(dsm(base(false, k - 1), chunk(k - 1)), lv.w[k - 1], lv.h[k - 1], i, j);
            d[t - R * c] = v; lv.down[k][t] = v;
        }
        cluster.sync();
    }
    for (int k = L - 2; k >= first; k--) {
        const int c = chunk(k), n = lv.w[k] * lv.h[k];
        float4* u = s_lv + base(true, k);
        const auto down = dsm(base(false, k), c);
        const auto coarse = dsm(k + 1 == L - 1 ? base(false, k + 1) : base(true, k + 1), chunk(k + 1));
        for (int t = R * c + threadIdx.x; t < min(n, (R + 1) * c); t += BLOOM_TAIL_THREADS) {
            const int j = t / lv.w[k], i = t - j * lv.w[k];
            const float4 v = bloom_up_at(down, coarse, lv.w[k], lv.w[k + 1], lv.h[k + 1], i, j, a);
            u[t - R * c] = v; lv.up[k][t] = v;
        }
        cluster.sync();
    }
}
#endif
// The Rgba8UnormSrgb store with the glow: x is what k_output_rgba8 (OP 0) or k_output_display<OP> would store before T, B = tent(up_0)
template <int OP>
__global__ void __launch_bounds__(ST_BLOCK) k_output_bloom(KPARAMS, uchar4* __restrict__ out, const u32* __restrict__ state, ExposureDev ep, BloomDev bp,
                                                           const float4* __restrict__ up0, int w0, int h0) {
    Px p = pixel_full(cam);
    if (!p.in) return;
    size_t i = pix(cam, p.x, p.y);
    const float4 c = cam.output[i];
    float3 x = f3(c.x, c.y, c.z);
    if (OP != 0) {
        const float ev = state ? __uint_as_float(state[0]) : ep.ev;
        const float s = pow_det(2.0f, ep.compensation - ev);
        x = f3((c.x > 0.0f ? c.x : 0.0f) * s, (c.y > 0.0f ? c.y : 0.0f) * s, (c.z > 0.0f ? c.z : 0.0f) * s);
    }
    const float4 B = bloom_tent(up0, w0, h0, (int)p.x, (int)p.y);
    const float I = bp.intensity;
    if (bp.mode == 0) { const float k = 1.0f - I; x = f3(x.x * k + B.x * I, x.y * k + B.y * I, x.z * k + B.z * I); }
    else x = f3(x.x + B.x * I, x.y + B.y * I, x.z + B.z * I);
    const float3 t = expo_transform<OP>(x);
    float v[3] = {t.x, t.y, t.z};
    u32 q[3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        float y = sat(v[k]);
        float e = (y <= 0.0031308f) ? 12.92f * y : 1.055f * pow_det(y, 1.0f / 2.4f) - 0.055f;
        q[k] = to_u32_sat(sat(e) * 255.0f + 0.5f);
    }
    out[i] = make_uchar4((unsigned char)q[0], (unsigned char)q[1], (unsigned char)q[2], 255);
}

// ---- Depth of field (ST_OPT_DEPTH_OF_FIELD; DESIGN.md §2 "Depth of field") ---------------------------------------------------------
// The gather stages each gathering tile's colours and radii, with a halo of its radius, in shared memory while the frame's max_radius
// is at most ST_DOF_STAGE_MAX_RADIUS, and reads every tap from global memory (L1 / L2) above it, where the stage (up to 80^2 texels,
// 128 KB at R = 32) leaves one CTA per SM: measured on an H100, the stage is faster at R = 16 and twice as slow at R = 32 (DESIGN.md
// §4).  Both read the same values: the words are the same (tools/depth_of_field_variants.py builds 0 and 32 as tuning builds).
#ifndef ST_DOF_STAGE_MAX_RADIUS
#define ST_DOF_STAGE_MAX_RADIUS 16
#endif
#define DOF_THREADS (kDofTile * kDofTile)
// r = clamp(k (z - F) / z, -R, R) with z = t dot(d, forward); the sky (t = 0) takes its limit min(k, R)
ST_DEV float dof_coc(const DofDev& p, float t, float3 d) {
    if (!p.active) return 0.0f;
    if (t == 0.0f) return p.k < p.R ? p.k : p.R;
    const float z = t * ((d.x * p.fwd_x + d.y * p.fwd_y) + d.z * p.fwd_z);
    const float r = p.k * (z - p.F) / z;
    return r < -p.R ? -p.R : (r > p.R ? p.R : r);
}
ST_DEV float dof_finite(float v) { return fabsf(v) < __int_as_float(0x7f800000) ? v : 0.0f; }
// One tap's weight: s = min(|r_q|, |r_p|) for a tap behind p (r_q > r_p: r increases with z), |r_q| otherwise;
// w = clamp(s - delta + 1, 0, 1) / max(s, 1/2)^2
ST_DEV float dof_weight(float rq, float rp, float delta) {
    const float aq = fabsf(rq), ap = fabsf(rp);
    const float s = rq > rp ? (aq < ap ? aq : ap) : aq;
    float c = (s - delta) + 1.0f;
    c = c < 0.0f ? 0.0f : (c > 1.0f ? 1.0f : c);
    const float m = s > 0.5f ? s : 0.5f;
    return c / (m * m);
}
// The gathered value of a pixel with radius rp, over the taps of radius rho; tap(dx, dy, &c, &r) reads the clamped neighbour
template <class T>
ST_DEV float4 dof_gather_px(const DofTap* __restrict__ taps, int rho, float rp, T tap) {
    const DofTap* row = taps + (size_t)(rho - 1) * kDofTaps;
    float ax = 0.0f, ay = 0.0f, az = 0.0f, ws = 0.0f;
    for (int i = 0; i < kDofTaps; i++) {
        const DofTap t = row[i];
        float4 c; float rq;
        tap((int)t.dx, (int)t.dy, &c, &rq);
        const float w = dof_weight(rq, rp, t.d);
        ax = ax + c.x * w; ay = ay + c.y * w; az = az + c.z * w; ws = ws + w;
    }
    return f4(ax / ws, ay / ws, az / ws, 1.0f);
}
// One CTA per 16 x 16 tile: every pixel's r, and the tile's max |r|; CTA (0, 0) writes the header words
__global__ void __launch_bounds__(DOF_THREADS) k_dof_coc(const __grid_constant__ CameraDev cam, const __grid_constant__ DofDev p, float* __restrict__ words,
                                                         float* __restrict__ tile_m) {
    __shared__ float s_m[DOF_THREADS / 32];
    const int x = blockIdx.x * kDofTile + threadIdx.x % kDofTile, y = blockIdx.y * kDofTile + threadIdx.x / kDofTile;
    float a = 0.0f;
    if (x < cam.w && y < cam.h) {
        const size_t i = (size_t)y * cam.w + x;
        const float r = dof_coc(p, cam.surface_nd[i].w, cam_ray(cam.curr, (u32)x, (u32)y).d);
        words[kDofHeaderWords + i] = r;
        a = fabsf(r);
    }
    for (int o = 16; o > 0; o >>= 1) { const float b = __shfl_xor_sync(0xffffffffu, a, o); a = a > b ? a : b; }
    if ((threadIdx.x & 31) == 0) s_m[threadIdx.x >> 5] = a;
    __syncthreads();
    if (threadIdx.x == 0) {
        float m = s_m[0];
        for (int k = 1; k < DOF_THREADS / 32; k++) m = m > s_m[k] ? m : s_m[k];
        tile_m[blockIdx.y * gridDim.x + blockIdx.x] = m;
    }
    if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x < kDofHeaderWords) words[threadIdx.x] = __uint_as_float(p.head[threadIdx.x]);
}
// One CTA per tile: rho_t = 0 when the largest max |r| of the tiles within `reach` is below 1/2 (the tile is copied), ceil of it
// otherwise; then each pixel's gather, from the shared-memory stage (STAGE) or from global memory
template <bool STAGE>
__global__ void __launch_bounds__(DOF_THREADS) k_dof_gather(const float4* __restrict__ output, int W, int H, const __grid_constant__ DofDev p,
                                                            float* __restrict__ words, const float* __restrict__ tile_m, const DofTap* __restrict__ taps,
                                                            float4* __restrict__ dof) {
    __shared__ int s_rho;
    const int tx = blockIdx.x, ty = blockIdx.y, TX = gridDim.x, TY = gridDim.y;
    if (threadIdx.x < 32) {   // the (2 reach + 1)^2 <= 25 neighbouring tiles, one per lane
        const int n = 2 * p.reach + 1, k = threadIdx.x;
        const int ux = tx - p.reach + k % n, uy = ty - p.reach + k / n;
        float m = (k < n * n && ux >= 0 && uy >= 0 && ux < TX && uy < TY) ? tile_m[uy * TX + ux] : 0.0f;
        for (int o = 16; o > 0; o >>= 1) { const float b = __shfl_xor_sync(0xffffffffu, m, o); m = m > b ? m : b; }
        if (k == 0) {
            const int rho = m < 0.5f ? 0 : (int)ceilf(m);
            s_rho = rho;
            words[kDofHeaderWords + (size_t)W * H + ty * TX + tx] = __uint_as_float((u32)rho);
        }
    }
    __syncthreads();
    const int rho = s_rho;
    const int lx = threadIdx.x % kDofTile, ly = threadIdx.x / kDofTile, x = tx * kDofTile + lx, y = ty * kDofTile + ly;
    const float* r = words + kDofHeaderWords;
    if (rho == 0) {   // nothing here is blurred: the frame is copied bit for bit
        if (x < W && y < H) dof[(size_t)y * W + x] = output[(size_t)y * W + x];
        return;
    }
    auto cx = [&](int v) { return v < 0 ? 0 : (v > W - 1 ? W - 1 : v); };
    auto cy = [&](int v) { return v < 0 ? 0 : (v > H - 1 ? H - 1 : v); };
    if (STAGE) {
        extern __shared__ float4 s_c[];   // (16 + 2 rho)^2 colours (non-finite channels read 0), then as many radii
        const int S = kDofTile + 2 * rho, x0 = tx * kDofTile - rho, y0 = ty * kDofTile - rho;
        float* s_r = (float*)(s_c + S * S);
        for (int k = threadIdx.x; k < S * S; k += DOF_THREADS) {
            const int sy = k / S, sx = k - sy * S;
            const size_t i = (size_t)cy(y0 + sy) * W + cx(x0 + sx);
            const float4 c = output[i];
            s_c[k] = f4(dof_finite(c.x), dof_finite(c.y), dof_finite(c.z), 0.0f);
            s_r[k] = r[i];
        }
        __syncthreads();
        if (x >= W || y >= H) return;
        const int c0 = (ly + rho) * S + lx + rho;
        dof[(size_t)y * W + x] = dof_gather_px(taps, rho, s_r[c0], [&](int dx, int dy, float4* c, float* rq) {
            const int k = c0 + dy * S + dx; *c = s_c[k]; *rq = s_r[k];
        });
        return;
    }
    if (x >= W || y >= H) return;
    dof[(size_t)y * W + x] = dof_gather_px(taps, rho, r[(size_t)y * W + x], [&](int dx, int dy, float4* c, float* rq) {
        const size_t i = (size_t)cy(y + dy) * W + cx(x + dx);
        const float4 v = ldg4(output + i);
        *c = f4(dof_finite(v.x), dof_finite(v.y), dof_finite(v.z), 0.0f); *rq = __ldg(r + i);
    });
}

// The thin-lens primary ray of pixel (x, y): a uniform point u of the unit disc, drawn by rejection from pairs of the lens stream (at
// most 16 pairs, else the centre), the origin moved to o + (right (h u.x) + up (h u.y)), aimed at the pinhole ray's point at view
// depth F, P_F = o + d (F / dot(d, fwd))
ST_DEV Ray lens_ray(const GpuCamera& c, const LensDev& l, u32 x, u32 y) {
    const Ray pin = cam_ray(c, x, y);
    Rng rng = rng_make(l.seed, x, y);
    float a = 0.0f, b = 0.0f;
    for (int i = 0; i < 16; i++) {
        const float u = rng_f(rng) * 2.0f - 1.0f, v = rng_f(rng) * 2.0f - 1.0f;
        if (u * u + v * v <= 1.0f) { a = u; b = v; break; }
    }
    const float ha = l.h * a, hb = l.h * b;
    const float3 o = pin.o + (f3(l.rx, l.ry, l.rz) * ha + f3(l.ux, l.uy, l.uz) * hb);
    const float s = l.F / ((pin.d.x * l.fx + pin.d.y * l.fy) + pin.d.z * l.fz);
    const float3 pf = pin.o + pin.d * s;
    return ray_make(o, norm(pf - o));
}
// K1 ref_tracing::main (ref_tracing.rs:4-60); NMAP: the packed normal is the mapped one, which K2 shades with and nudges along; LENS:
// the depth-0 ray is the thin-lens ray (ST_OPT_DEPTH_OF_FIELD)
template <bool NMAP, bool LENS>
__global__ void __launch_bounds__(ST_BLOCK) k_ref_tracing(KPARAMS, u32 depth, const __grid_constant__ LensDev lens) {
    ST_TRACE_STACK();
    Px p = pixel_full(cam);
    if (!p.in) return;
    size_t idx = screen_idx(cam, p.x, p.y);
    Ray ray;
    if (depth == 0u) ray = LENS ? lens_ray(cam.curr, lens, p.x, p.y) : cam_ray(cam.curr, p.x, p.y);
    else {
        float4 d0 = cam.ref_rays[3 * idx], d1 = cam.ref_rays[3 * idx + 1];
        if (all_zero(d1)) return;
        ray = ray_make(xyz(d0), xyz(d1));
    }
    TriHit h = trace_closest(ray, sc, stk);
    if (NMAP && trihit_some(h)) h.normal = nmap_normal(sc, h, ldg4(&sc.materials[h.material_id].normal_map_texture));
    float4 h0, h1; trihit_pack(h, &h0, &h1);
    cam.ref_hits[2 * idx] = h0; cam.ref_hits[2 * idx + 1] = h1;
}

// K2 ref_shading::main (ref_shading.rs:4-177); LGRID: the one light is drawn from the light grid's list for the nudged hit point
// TEXF: the hit's textures are filtered; the packed hit carries no triangle, so the segment's ray is traced again (same ray, same
// BVH: the same triangle and distance); ENVM: a path that leaves the scene sees the map; LENS: the depth-0 ray is K1's thin-lens ray
template <bool LGRID, bool TEXF, bool ENVM, bool LENS>
__global__ void __launch_bounds__(ST_BLOCK) k_ref_shading(KPARAMS, u32 seed, u32 depth, const __grid_constant__ LightGridDev lg,
                                                          const __grid_constant__ TexFilterDev tf, const __grid_constant__ EnvMapDev em,
                                                          const __grid_constant__ LensDev lens) {
    ST_TRACE_STACK();
    Px p = pixel_full(cam);
    if (!p.in) return;
    size_t idx = screen_idx(cam, p.x, p.y);
    Rng rng = rng_make(seed, p.x, p.y);
    float4* rays = cam.ref_rays;
    if (depth == 255u) {
        size_t i = pix(cam, p.x, p.y);
        float4 prev = cam_is_eq(cam.curr, cam.prev) ? cam.ref_colors[i] : f4zero();
        cam.ref_colors[i] = prev + f4(xyz(rays[3 * idx + 2]), 1.0f);
        return;
    }
    Ray ray; float3 color, thr;
    if (depth == 0u) { ray = LENS ? lens_ray(cam.curr, lens, p.x, p.y) : cam_ray(cam.curr, p.x, p.y); color = f3s(0.f); thr = f3s(1.0f); }
    else {
        float4 d0 = rays[3 * idx], d1 = rays[3 * idx + 1], d2 = rays[3 * idx + 2];
        if (all_zero(d1)) return;   // dead path: explicit no-op (the reference reaches the same state through 0 * x)
        ray = ray_make(xyz(d0), xyz(d1)); color = xyz(d2); thr = f3(d0.w, d1.w, d2.w);
    }
    TriHit th = trihit_unpack(cam.ref_hits[2 * idx], cam.ref_hits[2 * idx + 1]);
    if (!trihit_some(th)) {
        color = color + thr * sky_radiance<ENVM>(sc, em, world_sun_dir(sc.world), ray.d);
        rays[3 * idx] = f4zero(); rays[3 * idx + 1] = f4zero(); rays[3 * idx + 2] = f4(color, 0.0f);
        return;
    }
    GpuMaterial m = sc.materials[th.material_id];
    if (depth > 0u) m.roughness = rmax(m.roughness, 0.75f * 0.75f);
    Hit hit;
    hit.point = th.point + th.normal * 0.01f; hit.origin = ray.o; hit.dir = ray.d;
    if (TEXF) {
        const TriHit again = trace_closest(ray, sc, stk);
        uncount_ray(sc);
        TexFoot ft; ft.tri = again.triangle_id; ft.dir = ray.d; ft.w = texf_cone_width(cam.curr, p.x, p.y, again.t, depth == 0u);
        hit.g.base_color = texf_sample(sc, tf, th.material_id, 0u, m.base_color_texture, m.base_color, th.uv, ft);
        hit.g.emissive = xyz(texf_sample(sc, tf, th.material_id, 1u, m.emissive_texture, m.emissive, th.uv, ft));
    } else { hit.g.base_color = mat_base_color(sc, m, th.uv); hit.g.emissive = mat_emissive(sc, m, th.uv); }
    hit.g.normal = th.normal; hit.g.metallic = m.metallic;
    hit.g.roughness = m.roughness; hit.g.reflectance = m.reflectance; hit.g.depth = 0.0f;
    color = color + thr * hit.g.emissive;
    const LgList list = LGRID ? lgrid_list(lg, hit.point) : LgList{nullptr, sc.world.light_count};
    if (list.n > 0u) {
        u32 lid = lgrid_pick(list, rng_u32(rng) % list.n);
        float lpdf = 1.0f / (float)list.n;
        GpuLight light = light_load(sc, lid);
        bool occ = trace_any(light_ray_wnoise(light, rng, hit.point), sc, stk);
        if (!occ) color = color + thr * lightrad_sum(light_radiance(light, hit)) / lpdf;
    }
    BrdfS rs = brdf_layered_sample(hit.g, rng, -hit.dir);
    if (rs.pdf == 0.0f) { rays[3 * idx] = f4zero(); rays[3 * idx + 1] = f4zero(); return; }
    thr = thr * dot(rs.dir, hit.g.normal);
    thr = thr * (rs.radiance / rs.pdf);
    rays[3 * idx] = f4(hit.point, thr.x);
    rays[3 * idx + 1] = f4(rs.dir, thr.y);
    rays[3 * idx + 2] = f4(color, thr.z);
}

// K3 bvh_heatmap::main (bvh_heatmap.rs:4-77)
__global__ void __launch_bounds__(ST_BLOCK) k_bvh_heatmap(KPARAMS) {
    ST_TRACE_STACK();
    Px p = pixel_full(cam);
    if (!p.in) return;
    u32 used = 0u;
    trace_closest<true>(cam_ray(cam.curr, p.x, p.y), sc, stk, &used);
    float progress = (float)used / 8192.0f;
    const float3 cols[4] = {f3(0.f, 0.f, 1.f), f3(0.f, 1.f, 0.f), f3(1.f, 0.f, 0.f), f3(0.f, 0.f, 0.f)};
    float3 c = cols[3];
    if (progress <= 0.0f) c = cols[0];
    else {
        float step = 1.0f / (4.0f - 1.0f);
        bool done = false;
        for (int k = 0; k < 3 && !done; k++) {
            float mn = step * (float)k, mx = step * ((float)k + 1.0f);
            if (progress >= mn && progress <= mx) { float rhs = (progress - mn) / step; float lhs = 1.0f - rhs; c = lhs * cols[k] + rhs * cols[k + 1]; done = true; }
        }
    }
    cam.ref_colors[pix(cam, p.x, p.y)] = f4(c, 1.0f);
}

// ---------------------------------------------------------------------------------------------
// Ray-stream kernels (the K1/K8/K16 shape without the screen): 8 floats per ray
// (origin.xyz, len, dir.xyz, pad) in, packed hits / occlusion flags out.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(ST_BLOCK) k_trace_stream_closest(const __grid_constant__ SceneDev sc, const float4* __restrict__ rays, long n, float4* __restrict__ out) {
    ST_TRACE_STACK();
    long i = (long)blockIdx.x * ST_BLOCK + threadIdx.x;
    if (i >= n) return;
    float4 a = rays[2 * i], b = rays[2 * i + 1];
    u32 used = 0u;
    TriHit h = trace_closest<true>(ray_make(xyz(a), xyz(b)), sc, stk, &used);
    float4 h0, h1; trihit_pack(h, &h0, &h1);
    out[3 * i] = h0; out[3 * i + 1] = h1; out[3 * i + 2] = f4(h.t, bitsf(h.triangle_id), bitsf(h.material_id), (float)used);
}
__global__ void __launch_bounds__(ST_BLOCK) k_trace_stream_any(const __grid_constant__ SceneDev sc, const float4* __restrict__ rays, long n, u32* __restrict__ out) {
    ST_TRACE_STACK();
    long i = (long)blockIdx.x * ST_BLOCK + threadIdx.x;
    if (i >= n) return;
    float4 a = rays[2 * i], b = rays[2 * i + 1];
    out[i] = trace_any(ray_make(xyz(a), xyz(b), a.w), sc, stk) ? 1u : 0u;
}
// elementary-function test hook
__global__ void k_math(int op, const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out, long n) {
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float r = 0.f;
    switch (op) {
        case 0: r = sin_det(a[i]); break; case 1: r = cos_det(a[i]); break; case 2: r = acos_det(a[i]); break;
        case 3: r = atan2_det(a[i], b[i]); break; case 4: r = exp_det(a[i]); break; case 5: r = pow_det(a[i], b[i]); break;
        case 6: r = acos_approx_glam(a[i]); break;
    }
    out[i] = r;
}
// st_device_math op 7: the level of detail's log2 (ST_OPT_TEXTURE_FILTER)
__global__ void k_math_log2(const float* __restrict__ a, float* __restrict__ out, long n) {
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = log2_x(a[i]);
}
// st_device_math ops 8 and 9: the environment map's acos and atan2(a, b)
__global__ void k_math_envm(int op, const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out, long n) {
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = op == 8 ? acos_x(a[i]) : atan2_x(a[i], b[i]);
}

// ST_OPT_TEXTURE_FILTER: level k+1 of the images of `jobs` (blockIdx.y) from their level k, one thread per output texel.  Texel (x, y)
// averages level-k texels (min(2x + i, w - 1), min(2y + j, h - 1)), i, j in {0, 1}: r, g, b decoded through the sRGB table, summed
// ((c00 + c10) + c01) + c11, times 0.25, re-encoded to the byte whose table value is nearest (ties to the lower byte: the count of the
// 255 midpoints below the value); alpha (a00 + a10 + a01 + a11 + 2) >> 2.
__global__ void __launch_bounds__(256) k_texture_mips(const MipJob* __restrict__ jobs, const uchar4* __restrict__ atlas, uchar4* __restrict__ pool,
                                                      const float* __restrict__ srgb) {
    __shared__ float lut[256], mid[255];
    lut[threadIdx.x] = srgb[threadIdx.x];
    __syncthreads();
    if (threadIdx.x < 255u) mid[threadIdx.x] = xmul(xadd(lut[threadIdx.x], lut[threadIdx.x + 1u]), 0.5f);
    __syncthreads();
    const MipJob j = jobs[blockIdx.y];
    const u32 i = blockIdx.x * 256u + threadIdx.x;
    if (i >= j.dst_w * j.dst_h) return;
    const u32 x = i % j.dst_w, y = i / j.dst_w;
    const u32 xa = min(2u * x, j.src_w - 1u), xb = min(2u * x + 1u, j.src_w - 1u), ya = min(2u * y, j.src_h - 1u), yb = min(2u * y + 1u, j.src_h - 1u);
    const uchar4* src = (j.from_atlas ? atlas : pool) + j.src;
    const size_t st = j.src_stride;
    const uchar4 c00 = src[ya * st + xa], c10 = src[ya * st + xb], c01 = src[yb * st + xa], c11 = src[yb * st + xb];
    const u32 b0[3] = {c00.x, c00.y, c00.z}, b1[3] = {c10.x, c10.y, c10.z}, b2[3] = {c01.x, c01.y, c01.z}, b3[3] = {c11.x, c11.y, c11.z};
    u32 out[3];
#pragma unroll
    for (int c = 0; c < 3; c++) {
        const float s = xmul(xadd(xadd(xadd(lut[b0[c]], lut[b1[c]]), lut[b2[c]]), lut[b3[c]]), 0.25f);
        u32 b = 0u;
        for (u32 step = 128u; step > 0u; step >>= 1) if (b + step <= 255u && mid[b + step - 1u] < s) b += step;
        out[c] = b;
    }
    const u32 a = ((u32)c00.w + (u32)c10.w + (u32)c01.w + (u32)c11.w + 2u) >> 2;
    pool[j.dst + i] = make_uchar4((unsigned char)out[0], (unsigned char)out[1], (unsigned char)out[2], (unsigned char)a);
}

// ST_OPT_LIGHT_GRID: the candidate lists (DESIGN.md §2 "Light grid").  One warp per cell, the outside list last (cell == ncell: no
// cell box, so only the non-cullable slots).  The warp tests 32 slots at a time and compacts the kept ones with ballot / popc in
// ascending slot order: deterministic with no sort and no atomics.  A cullable light is dropped when the squared distance from its
// centre to the cell box grown by `margin` exceeds range^2 (1 + 2^-8); the entries past the count are 0xffffffff.
__global__ void __launch_bounds__(128) k_light_grid_build(const __grid_constant__ LightGridDev lg, const GpuLight* __restrict__ lights, u32 ncell,
                                                          u32* __restrict__ counts, u32* __restrict__ lists) {
    const u32 lane = threadIdx.x & 31u, cell = blockIdx.x * 4u + (threadIdx.x >> 5);
    if (cell > ncell) return;   // whole warps
    const bool outside = cell == ncell;
    float bmin[3] = {0.f, 0.f, 0.f}, bmax[3] = {0.f, 0.f, 0.f};
    if (!outside) {
        const u32 idx[3] = {cell % lg.dims[0], (cell / lg.dims[0]) % lg.dims[1], cell / (lg.dims[0] * lg.dims[1])};
        for (int a = 0; a < 3; a++) {
            bmin[a] = xsub(xadd(lg.lo[a], xmul((float)idx[a], lg.cell[a])), lg.margin[a]);
            bmax[a] = xadd(xadd(lg.lo[a], xmul((float)(idx[a] + 1u), lg.cell[a])), lg.margin[a]);
        }
    }
    u32* out = lists + (size_t)cell * kLightGridK;
    u32 n = 0u;
    for (u32 base = 0u; base < lg.light_count; base += 32u) {
        const u32 slot = base + lane;
        bool keep = false;
        if (slot < lg.light_count) {
            const float4* p = reinterpret_cast<const float4*>(lights + slot);
            GpuLight l; l.d0 = ldg4(p); l.d1 = ldg4(p + 1); l.d2 = ldg4(p + 2);
            if (!lgrid_cullable(l)) keep = true;
            else if (!outside) {
                const float c[3] = {l.d0.x, l.d0.y, l.d0.z};
                float d[3];
                for (int a = 0; a < 3; a++) d[a] = fmaxf(fmaxf(xsub(bmin[a], c[a]), xsub(c[a], bmax[a])), 0.0f);
                const float d2 = xadd(xadd(xmul(d[0], d[0]), xmul(d[1], d[1])), xmul(d[2], d[2]));
                keep = !(d2 > xmul(xmul(l.d1.w, l.d1.w), 1.00390625f));
            }
        }
        const u32 mask = __ballot_sync(0xffffffffu, keep);
        const u32 pos = n + __popc(mask & ((1u << lane) - 1u));
        if (keep && pos < kLightGridK) out[pos] = slot;
        n += __popc(mask);
    }
    for (u32 k = min(n, kLightGridK) + lane; k < kLightGridK; k += 32u) out[k] = 0xffffffffu;
    if (lane == 0u) counts[cell] = n > kLightGridK ? kLightGridOverflow : n;
}

// derived tables: packed gamma colour per material, byte -> linear table for GBufferEntry::unpack
__global__ void k_material_derive(const GpuMaterial* __restrict__ mats, u32 n, u32* __restrict__ packed) {
    u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) packed[i] = gbuf_pack_color(mats[i].base_color);
}
__global__ void k_srgb_lut(float* __restrict__ lut) {   // sRGB electro-optical transfer function per byte
    u32 i = threadIdx.x;
    float c = (float)i / 255.0f;
    lut[i] = (c <= 0.04045f) ? c / 12.92f : pow_det((c + 0.055f) / 1.055f, 2.4f);
}
__global__ void k_unpack_lut(float* __restrict__ lut) {
    u32 i = threadIdx.x;   // 256 threads
    lut[i] = pow_det((float)i / 255.0f, 2.2f);
    lut[256u + i] = pow_det((float)i / 63.0f, 2.2f);
}

// ---------------------------------------------------------------------------------------------
// Atmosphere LUT generation (strolle-shaders/src/atmosphere/*.rs; Hillaire 2020).  Runs once /
// on sun change (90 k texels) — outside the per-frame hot path, kept on the GPU so that the
// product needs no CPU fallback for it.  Rgba16Float storage == f32 rounded to binary16.
// ---------------------------------------------------------------------------------------------
ST_DEV float round_f16(float f) { return __half2float(__float2half_rn(f)); }
ST_DEV void atm_scattering(float3 pos, float3* rayleigh, float* mie, float3* ext) {   // atmosphere/utils.rs:3-27
    float alt_km = (len(pos) - ST_ATM_GROUND) * 1000.0f;
    float rd = exp_det(-alt_km / 8.0f);
    float md = exp_det(-alt_km / 1.2f);
    float3 rs = f3(5.802f, 13.558f, 33.1f) * rd;
    float ms = 3.996f * md;
    float ma = 4.4f * md;
    float3 oz = f3(0.650f, 1.881f, 0.085f) * rmax(1.0f - fabs_(alt_km - 25.0f) / 15.0f, 0.0f);
    *rayleigh = rs; *mie = ms;
    *ext = ((rs + f3s(ms)) + f3s(ma)) + oz;   // RAYLEIGH_ABSORPTION_BASE == 0.0 contributes nothing (quirk C-18)
}
ST_DEV float atm_mie_phase(float c) {
    const float G = 0.8f; const float SCALE = 3.0f / (8.0f * kPi);
    float num = (1.0f - G * G) * (1.0f + c * c);
    float den = (2.0f + G * G) * pow_det(1.0f + G * G - 2.0f * G * c, 1.5f);
    return SCALE * num / den;
}
ST_DEV float atm_rayleigh_phase(float c) { const float K = 3.0f / (16.0f * kPi); return K * (1.0f + c * c); }
ST_DEV float3 exp3(float3 v) { return f3(exp_det(v.x), exp_det(v.y), exp_det(v.z)); }
ST_DEV float3 atm_transmittance(float3 pos, float3 sun_dir) {   // generate_transmittance_lut.rs:29-59
    if (ray_sphere(ray_make(pos, sun_dir), ST_ATM_GROUND) > 0.0f) return f3s(0.f);
    float adist = ray_sphere(ray_make(pos, sun_dir), ST_ATM_TOP);
    float t = 0.0f; float3 tr = f3s(1.0f);
    for (float i = 0.0f; i < 40.0f; i += 1.0f) {
        float nt = ((i + 0.3f) / 40.0f) * adist;
        float dt = nt - t; t = nt;
        float3 rs, ext; float ms; atm_scattering(pos + t * sun_dir, &rs, &ms, &ext);
        tr = tr * exp3(-dt * ext);
    }
    return tr;
}
__global__ void k_atm_transmittance(float4* __restrict__ out) {   // 256x64
    int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= 256 || y >= 64) return;
    float2 uv = f2((float)x, (float)y) / f2(256.0f, 64.0f);
    float sct = 2.0f * uv.x - 1.0f;
    float sth = acos_det(rclamp(sct, -1.0f, 1.0f));
    float height = lerpc(ST_ATM_GROUND, ST_ATM_TOP, uv.y);
    float3 v = atm_transmittance(f3(0.0f, height, 0.0f), norm(f3(0.0f, sct, -sin_det(sth))));
    out[y * 256 + x] = f4(round_f16(v.x), round_f16(v.y), round_f16(v.z), 1.0f);
}
__global__ void k_atm_sun_color(float4* __restrict__ out, GpuWorld world) {   // strolle/src/lights.rs:84-99
    float3 sd = world_sun_dir(world);
    float3 c = atm_transmittance(atm_view_pos(), sd);
    c = c * 20.0f * 5.0f;
    float3 pos = sd * 1000.0f;
    out[0] = f4(pos, 25.0f); out[1] = f4(c, finf());
}
__global__ void k_atm_scattering(const float4* __restrict__ tl, float4* __restrict__ out) {   // 32x32, generate_scattering_lut.rs
    int x = threadIdx.x, y = blockIdx.x;
    float2 uv = f2((float)x, (float)y) / f2(32.0f, 32.0f);
    float sct = 2.0f * uv.x - 1.0f;
    float sth = acos_det(rclamp(sct, -1.0f, 1.0f));
    float height = lerpc(ST_ATM_GROUND, ST_ATM_TOP, rmax(uv.y, 0.01f));
    float3 pos = f3(0.0f, height, 0.0f);
    float3 sun_dir = norm(f3(0.0f, sct, -sin_det(sth)));
    float3 lum_total = f3s(0.f), fms = f3s(0.f);
    const int S = 8;
    float inv_samples = 1.0f / (float)(S * S);
    for (int i = 0; i < S; i++) for (int j = 0; j < S; j++) {
        float theta = kPi * ((float)i + 0.5f) / (float)S;
        float phi = acos_det(rclamp(1.0f - 2.0f * ((float)j + 0.5f) / (float)S, -1.0f, 1.0f));
        float sph, cph, sth2, cth2; sincos_det(phi, &sph, &cph); sincos_det(theta, &sth2, &cth2);
        float3 rd = f3(sph * sth2, cph, sph * cth2);
        float adist = ray_sphere(ray_make(pos, rd), ST_ATM_TOP);
        float gdist = ray_sphere(ray_make(pos, rd), ST_ATM_GROUND);
        float t_max = (gdist > 0.0f) ? gdist : adist;
        float ct = dot(rd, sun_dir);
        float mp = atm_mie_phase(ct), rp = atm_rayleigh_phase(-ct);
        float3 lum = f3s(0.f), lf = f3s(0.f), tr = f3s(1.0f);
        float t = 0.0f;
        for (float s = 0.0f; s < 20.0f; s += 1.0f) {
            float nt = ((s + 0.3f) / 20.0f) * t_max;
            float dt = nt - t; t = nt;
            float3 np = pos + t * rd;
            float3 rs, ext; float ms; atm_scattering(np, &rs, &ms, &ext);
            float3 st_ = exp3(-dt * ext);
            float3 snp = rs + f3s(ms);
            float3 sf = (snp - snp * st_) / ext;
            lf = lf + tr * sf;
            float3 sun_t = atm_lut(tl, 256, 64, np, sun_dir);
            float3 ri = rs * rp;
            float mi = ms * mp;
            float3 ins = (ri + f3s(mi)) * sun_t;
            float3 si = (ins - ins * st_) / ext;
            lum = lum + si * tr;
            tr = tr * st_;
        }
        if (gdist > 0.0f) {
            float3 hp = pos + gdist * rd;
            if (dot(pos, sun_dir) > 0.0f) {
                hp = norm(hp) * ST_ATM_GROUND;
                lum = lum + tr * f3s(0.25f) * atm_lut(tl, 256, 64, hp, sun_dir);
            }
        }
        fms = fms + lf * inv_samples;
        lum_total = lum_total + lum * inv_samples;
    }
    float3 o = lum_total / (f3s(1.0f) - fms);
    out[y * 32 + x] = f4(round_f16(o.x), round_f16(o.y), round_f16(o.z), 1.0f);
}
__global__ void k_atm_sky(const float4* __restrict__ tl, const float4* __restrict__ sl, float sun_altitude, float4* __restrict__ out) {   // 256x256, generate_sky_lut.rs
    int x = threadIdx.x, y = blockIdx.x;
    float2 uv = f2((float)x, (float)y) / f2(256.0f, 256.0f);
    float azimuth = (uv.x - 0.5f) * 2.0f * kPi;
    float v;
    if (uv.y < 0.5f) { float c = 1.0f - 2.0f * uv.y; v = -c * c; }
    else { float c = uv.y * 2.0f - 1.0f; v = c * c; }
    float3 vp = atm_view_pos();
    float height = len(vp);
    float horizon;
    { float t = sq(height) - sq(ST_ATM_GROUND); t = sqrtf(t) / height; horizon = acos_det(rclamp(t, -1.0f, 1.0f)) - 0.5f * kPi; }
    float altitude = v * 0.5f * kPi - horizon;
    float sa, ca, sz, cz; sincos_det(altitude, &sa, &ca); sincos_det(azimuth, &sz, &cz);
    float3 rd = f3(ca * sz, sa, -ca * cz);
    float sal = fmodf(sun_altitude, 2.0f * kPi);
    float ss, cs_; sincos_det(sal, &ss, &cs_);
    float3 sun_dir = (sal < 0.5f * kPi) ? f3(0.0f, ss, -cs_) : f3(0.0f, ss, cs_);
    float adist = ray_sphere(ray_make(vp, rd), ST_ATM_TOP);
    float gdist = ray_sphere(ray_make(vp, rd), ST_ATM_GROUND);
    float t_max = (gdist < 0.0f) ? adist : gdist;
    float ct = dot(rd, sun_dir);
    float mp = atm_mie_phase(ct), rp = atm_rayleigh_phase(-ct);
    float3 lum = f3s(0.f), tr = f3s(1.0f);
    float t = 0.0f;
    for (float i = 0.0f; i < 32.0f; i += 1.0f) {
        float nt = ((i + 0.3f) / 32.0f) * t_max;
        float dt = nt - t; t = nt;
        float3 np = vp + t * rd;
        float3 rs, ext; float ms; atm_scattering(np, &rs, &ms, &ext);
        float3 st_ = exp3(-dt * ext);
        float3 sun_t = atm_lut(tl, 256, 64, np, sun_dir);
        float3 psi = atm_lut(sl, 32, 32, np, sun_dir);
        float3 ri = rs * (rp * sun_t + psi);
        float3 mi = ms * (mp * sun_t + psi);
        float3 ins = ri + mi;
        float3 si = (ins - ins * st_) / ext;
        lum = lum + si * tr;
        tr = tr * st_;
    }
    out[y * 256 + x] = f4(round_f16(lum.x), round_f16(lum.y), round_f16(lum.z), 1.0f);
}

#endif   // ST_EXACT_ONLY

// elementary-function test hook for the shading kernels' own flavour: in the fast build these are the SFU / approximate forms
// (sincos_det = __sincosf, exp_det = __expf, pow_det = __powf outside its product exponents, sqrtf = sqrt.approx, a / b = div.full)
__global__ void k_math_shading(int op, const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out, long n) {
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float r = 0.f, x = a[i], y = b[i];
    switch (op) {
        case 0: r = sin_det(x); break; case 1: r = cos_det(x); break; case 2: r = exp_det(x); break;
        case 3: r = pow_det(x, y); break; case 4: r = sqrtf(x); break; case 5: r = x / y; break;
        case 6: r = acos_det(x); break; case 7: r = atan2_det(x, y); break;
    }
    out[i] = r;
}

// ---------------------------------------------------------------------------------------------
// Host-side launchers
// ---------------------------------------------------------------------------------------------
static dim3 grid_full(const CameraDev& cam) { return dim3((cam.w + TILE_W - 1) / TILE_W, (cam.y1 - cam.y0 + TILE_H - 1) / TILE_H); }
static dim3 grid_half(const CameraDev& cam) { int hw = 8 * (((cam.w + 7) / 8) / 2); return dim3((hw + TILE_W - 1) / TILE_W, (cam.y1 - cam.y0 + TILE_H - 1) / TILE_H); }
#define HALF_LAUNCH(kernel, c, st, ...) do { dim3 g_ = grid_half(c); if (g_.x > 0 && g_.y > 0) kernel<<<g_, ST_BLOCK, 0, st>>>(__VA_ARGS__); } while (0)

void launch_di_sampling(const CameraDev& c, const SceneDev& s, int cur, u32 seed, u32 frame, const LightGridDev* lg, cudaStream_t st) {
    if (lg) k_di_sampling<true><<<grid_full(c), ST_BLOCK, 0, st>>>(c, s, cur, seed, frame, *lg); else k_di_sampling<false><<<grid_full(c), ST_BLOCK, 0, st>>>(c, s, cur, seed, frame, LightGridDev{});
}
void launch_di_temporal(const CameraDev& c, const SceneDev& s, int cur, u32 seed, cudaStream_t st) { k_di_temporal<<<grid_full(c), ST_BLOCK, 0, st>>>(c, s, cur, seed); }
void launch_di_spatial_pick(const CameraDev& c, const SceneDev& s, int cur, u32 seed, u32 frame, cudaStream_t st) { HALF_LAUNCH(k_di_spatial_pick, c, st, c, s, cur, seed, frame); }
void launch_spatial_trace(const CameraDev& c, const SceneDev& s, const float4* d0, const float4* d1, float4* d2, cudaStream_t st) { k_spatial_trace<<<grid_full(c), ST_BLOCK, 0, st>>>(c, s, d0, d1, d2); }
void launch_di_spatial_sample(const CameraDev& c, const SceneDev& s, u32 seed, u32 frame, cudaStream_t st) { HALF_LAUNCH(k_di_spatial_sample, c, st, c, s, seed, frame); }
void launch_di_resolving(const CameraDev& c, const SceneDev& s, int cur, const EnvMapDev* em, cudaStream_t st) {
    if (em) k_di_resolving<true><<<grid_full(c), ST_BLOCK, 0, st>>>(c, s, cur, *em); else k_di_resolving<false><<<grid_full(c), ST_BLOCK, 0, st>>>(c, s, cur, EnvMapDev{});
}
void launch_gi_reprojection(const CameraDev& c, const SceneDev& s, int cur, cudaStream_t st) { k_gi_reprojection<<<grid_full(c), ST_BLOCK, 0, st>>>(c, s, cur); }
void launch_gi_sampling_a(const CameraDev& c, const SceneDev& s, int cur, u32 seed, u32 frame, bool nmap, const TexFilterDev* tf, const EnvMapDev* em,
                          cudaStream_t st) {
    const TexFilterDev tnone{};
    const TexFilterDev& t = tf ? *tf : tnone;
    const EnvMapDev enone{};
    const EnvMapDev& m = em ? *em : enone;
#define ST_GSA(N_, T_, E_) HALF_LAUNCH((k_gi_sampling_a<N_, T_, E_>), c, st, c, s, cur, seed, frame, t, m)
#define ST_GSA_E(N_, T_) do { if (em && em->cdf) ST_GSA(N_, T_, ENV_SAMPLED); else ST_GSA(N_, T_, ENV_NONE); } while (0)
    if (tf) { if (nmap) ST_GSA_E(true, true); else ST_GSA_E(false, true); }
    else { if (nmap) ST_GSA_E(true, false); else ST_GSA_E(false, false); }
#undef ST_GSA_E
#undef ST_GSA
}
void launch_gi_sampling_b(const CameraDev& c, const SceneDev& s, int cur, u32 seed, u32 frame, const LightGridDev* lg, const EnvMapDev* em, cudaStream_t st) {
    const LightGridDev none{};
    const LightGridDev& g = lg ? *lg : none;
    const EnvMapDev enone{};
    const EnvMapDev& m = em ? *em : enone;
#define ST_GSB(L_, E_) HALF_LAUNCH((k_gi_sampling_b<L_, E_>), c, st, c, s, cur, seed, frame, g, m)
#define ST_GSB_E(L_) do { if (!em) ST_GSB(L_, ENV_NONE); else if (em->cdf) ST_GSB(L_, ENV_SAMPLED); else ST_GSB(L_, ENV_MAP); } while (0)
    if (lg) ST_GSB_E(true); else ST_GSB_E(false);
#undef ST_GSB_E
#undef ST_GSB
}
void launch_gi_temporal(const CameraDev& c, const SceneDev& s, int cur, u32 seed, u32 frame, int inline_reprojection, cudaStream_t st) { k_gi_temporal<<<grid_full(c), ST_BLOCK, 0, st>>>(c, s, cur, seed, frame, inline_reprojection); }
void launch_gi_spatial_pick(const CameraDev& c, const SceneDev& s, int cur, u32 seed, u32 frame, cudaStream_t st) { HALF_LAUNCH(k_gi_spatial_pick, c, st, c, s, cur, seed, frame); }
void launch_gi_spatial_sample(const CameraDev& c, const SceneDev& s, u32 seed, u32 frame, cudaStream_t st) { HALF_LAUNCH(k_gi_spatial_sample, c, st, c, s, seed, frame); }
void launch_gi_preview(const CameraDev& c, const SceneDev& s, int cur, u32 seed, u32 nth, const float4* in, float4* out, int mirror_reach, cudaStream_t st) { k_gi_preview<<<grid_full(c), ST_BLOCK, 0, st>>>(c, s, cur, seed, nth, in, out, mirror_reach); }
void launch_gi_resolving(const CameraDev& c, const SceneDev& s, int cur, const float4* in, cudaStream_t st) { k_gi_resolving<<<grid_full(c), ST_BLOCK, 0, st>>>(c, s, cur, in); }
void launch_di_sample_temporal(const CameraDev& c, const SceneDev& s, int cur, u32 seed_sampling, u32 seed_temporal, u32 frame, const LightGridDev* lg, cudaStream_t st) {
    if (lg) k_di_sample_temporal<true><<<grid_full(c), ST_BLOCK, 0, st>>>(c, s, cur, seed_sampling, seed_temporal, frame, *lg);
    else k_di_sample_temporal<false><<<grid_full(c), ST_BLOCK, 0, st>>>(c, s, cur, seed_sampling, seed_temporal, frame, LightGridDev{});
}
void launch_di_spatial_fused(const CameraDev& c, const SceneDev& s, int cur, u32 seed_pick, u32 seed_sample, u32 frame, cudaStream_t st) { HALF_LAUNCH(k_di_spatial_fused, c, st, c, s, cur, seed_pick, seed_sample, frame); }
void launch_gi_sampling_fused(const CameraDev& c, const SceneDev& s, int cur, u32 seed_a, u32 seed_b, u32 frame, bool nmap, const LightGridDev* lg, const TexFilterDev* tf,
                              const EnvMapDev* em, cudaStream_t st) {
    const LightGridDev none{};
    const LightGridDev& g = lg ? *lg : none;
    const TexFilterDev tnone{};
    const TexFilterDev& t = tf ? *tf : tnone;
    const EnvMapDev enone{};
    const EnvMapDev& m = em ? *em : enone;
#define ST_GSF(N_, L_, T_, E_) HALF_LAUNCH((k_gi_sampling_fused<N_, L_, T_, E_>), c, st, c, s, cur, seed_a, seed_b, frame, g, t, m)
#define ST_GSF_E(N_, L_, T_) do { if (!em) ST_GSF(N_, L_, T_, ENV_NONE); else if (em->cdf) ST_GSF(N_, L_, T_, ENV_SAMPLED); else ST_GSF(N_, L_, T_, ENV_MAP); } while (0)
    if (tf) {
        if (lg) { if (nmap) ST_GSF_E(true, true, true); else ST_GSF_E(false, true, true); }
        else { if (nmap) ST_GSF_E(true, false, true); else ST_GSF_E(false, false, true); }
    } else {
        if (lg) { if (nmap) ST_GSF_E(true, true, false); else ST_GSF_E(false, true, false); }
        else { if (nmap) ST_GSF_E(true, false, false); else ST_GSF_E(false, false, false); }
    }
#undef ST_GSF_E
#undef ST_GSF
}
void launch_gi_spatial_fused(const CameraDev& c, const SceneDev& s, int cur, u32 seed_pick, u32 seed_sample, u32 frame, cudaStream_t st) { HALF_LAUNCH(k_gi_spatial_fused, c, st, c, s, cur, seed_pick, seed_sample, frame); }
void launch_gi_preview_resolve(const CameraDev& c, const SceneDev& s, int cur, u32 seed, const float4* in, const float4* source, cudaStream_t st) { k_gi_preview_resolve<<<grid_full(c), ST_BLOCK, 0, st>>>(c, s, cur, seed, in, source); }
void launch_math_shading(int op, const float* a, const float* b, float* out, long n, cudaStream_t st) { k_math_shading<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(op, a, b, out, n); }
#if ST_EXACT_ONLY
void launch_prim_gbuffer(const CameraDev& c, const SceneDev& s, int cur, int with_reprojection, bool nmap, const TexFilterDev* tf, cudaStream_t st) {
    const TexFilterDev none{};
    const TexFilterDev& t = tf ? *tf : none;
#define ST_PG(N_, T_) k_prim_gbuffer<N_, T_><<<grid_full(c), ST_BLOCK, 0, st>>>(c, s, cur, with_reprojection, t)
    if (tf) { if (nmap) ST_PG(true, true); else ST_PG(false, true); }
    else { if (nmap) ST_PG(true, false); else ST_PG(false, false); }
#undef ST_PG
}
void launch_frame_reprojection(const CameraDev& c, const SceneDev& s, int cur, cudaStream_t st) { k_frame_reprojection<<<grid_full(c), ST_BLOCK, 0, st>>>(c, s, cur); }
void launch_denoise_reproject(const CameraDev& c, const SceneDev& s, int cur, const float4* pc, const float4* pm, const float4* smp, float4* col, float4* mom, cudaStream_t st) { k_denoise_reproject<<<grid_full(c), ST_BLOCK, 0, st>>>(c, s, cur, pc, pm, smp, col, mom); }
void launch_denoise_reproject_pair(const CameraDev& c, const SceneDev& s, int cur, cudaStream_t st) {
    ReprojectSignal di{c.di_diff_prev_colors, c.di_diff_moments[cur ^ 1], c.di_diff_samples, c.di_diff_curr_colors, c.di_diff_moments[cur]};
    ReprojectSignal gi{c.gi_diff_prev_colors, c.gi_diff_moments[cur ^ 1], c.gi_diff_samples, c.gi_diff_curr_colors, c.gi_diff_moments[cur]};
    k_denoise_reproject_pair<<<grid_full(c), ST_BLOCK, 0, st>>>(c, s, cur, di, gi);
}
void launch_denoise_variance(const CameraDev& c, const SceneDev& s, int cur, bool fast, cudaStream_t st) {
    if (fast) k_denoise_variance<true><<<grid_full(c), ST_BLOCK, 0, st>>>(c, s, cur); else k_denoise_variance<false><<<grid_full(c), ST_BLOCK, 0, st>>>(c, s, cur);
}
void launch_denoise_wavelet(const CameraDev& c, const SceneDev& s, int cur, u32 frame, u32 stride, float strength, const float4* di_in, float4* di_out, const float4* gi_in, float4* gi_out,
                            const float4* pair_in, float4* pair_out, bool fast, cudaStream_t st) {
#define ST_WG(F_, P_) k_denoise_wavelet<F_, P_><<<grid_full(c), ST_BLOCK, 0, st>>>(c, s, cur, frame, stride, strength, di_in, di_out, gi_in, gi_out, pair_in, pair_out)
    if (pair_in) { if (fast) ST_WG(true, true); else ST_WG(false, true); }
    else { if (fast) ST_WG(true, false); else ST_WG(false, false); }
#undef ST_WG
}
// K21, tile-staged: the 6x5 window of frame_denoising::estimate_variance (quirk C-3: row -2 spans x in [-2,2], rows -1..2 span
// x in [-3,2]) is only walked by pixels whose history is shorter than 4 frames, but a warp pays for it as soon as one of its
// pixels does; with the (TW+6) x (TH+4) neighbourhood in shared memory (three TMA tensor copies, zero fill outside the frame)
// those 29 taps are LDS.128 at fixed offsets instead of 87 gathered global loads.  Same taps, order and arithmetic as
// k_denoise_variance.
template <int TW, int TH> struct VarianceTile {
    static constexpr int HX = 3, HY = 2, BW = TW + 2 * HX, BH = TH + 2 * HY;
    static constexpr u32 BOX_BYTES = (u32)(BW * BH * 16);
    static constexpr u32 PLANE = (BOX_BYTES + 127u) & ~127u;
    static constexpr u32 SMEM = 3u * PLANE + 128u;
};
template <bool FAST, int TW, int TH>
__global__ void __launch_bounds__(TW * TH) k_denoise_variance_tiled(KPARAMS, int cur, const __grid_constant__ CUtensorMap tm_nd, const __grid_constant__ CUtensorMap tm_di,
                                                                    const __grid_constant__ CUtensorMap tm_gi, u32* __restrict__ errors) {
    typedef VarianceTile<TW, TH> T;
    extern __shared__ unsigned char s_raw[];
    __shared__ __align__(8) unsigned long long s_bar;
    const int tx = (int)threadIdx.x % TW, ty = (int)threadIdx.x / TW;
    const int x0 = (int)blockIdx.x * TW, y0 = cam.y0 + (int)blockIdx.y * TH;
    const u32 bar = smem_addr(&s_bar);
    const u32 raw = smem_addr(s_raw);
    const u32 base = (raw + 127u) & ~127u;
    if (threadIdx.x == 0) { mbar_init(bar, 1u); mbar_fence_init(); }
    __syncthreads();
    if (threadIdx.x == 0) {
        mbar_expect_tx(bar, 3u * T::BOX_BYTES);
        tma_load_2d(base, &tm_nd, (x0 - T::HX) * 2, y0 - T::HY, bar);
        tma_load_2d(base + T::PLANE, &tm_di, (x0 - T::HX) * 2, y0 - T::HY, bar);
        tma_load_2d(base + 2u * T::PLANE, &tm_gi, (x0 - T::HX) * 2, y0 - T::HY, bar);
    }
    const u32 px = (u32)(x0 + tx), py = (u32)(y0 + ty);
    const bool in = px < (u32)cam.w && py < (u32)cam.y1;
    const size_t i = in ? pix(cam, px, py) : 0;
    float4 mdi = f4zero(), mgi = f4zero();
    if (in) { mdi = cam.di_diff_moments[cur][i]; mgi = cam.gi_diff_moments[cur][i]; }   // in flight together with the tile
    {
        bool done = false;
        for (u32 spin = 0; spin < (1u << 20) && !done; spin++) done = mbar_try_wait(bar, 0u);
        if (!done) { if (threadIdx.x == 0) atomicAdd(errors, 1u); return; }
    }
    if (!in) return;
    const float4* __restrict__ t_nd = reinterpret_cast<const float4*>(s_raw + (base - raw));
    const float4* __restrict__ t_di = reinterpret_cast<const float4*>(s_raw + (base - raw) + T::PLANE);
    const float4* __restrict__ t_gi = reinterpret_cast<const float4*>(s_raw + (base - raw) + 2u * T::PLANE);
    const int c = (ty + T::HY) * T::BW + (tx + T::HX);
    float4 cnd = t_nd[c];
    float4 cdi = t_di[c], cgi = t_gi[c];
    if (cnd.w == 0.0f) { cam.di_diff_stash[i] = cdi; cam.gi_diff_stash[i] = cgi; return; }
    float di_var, gi_var;
    if (mdi.x >= 4.0f) { di_var = mdi.z - sq(mdi.y); gi_var = mgi.z - sq(mgi.y); }
    else {
        float3 cn = xyz(cnd);
        float scdl = sv_sqrt<FAST>(sv_luma<FAST>(xyz(cdi))), scgl = sv_sqrt<FAST>(sv_luma<FAST>(xyz(cgi)));
        float3 sdi = f3s(0.f), sgi = f3s(0.f);
#pragma unroll
        for (int oy = -2; oy <= 2; oy++) {
#pragma unroll
            for (int ox = -3; ox <= 2; ox++) {
                if (oy == -2 && ox == -3) continue;   // quirk C-3: the first row starts at -2
                const int k = c + oy * T::BW + ox;
                float4 nds = t_nd[k];
                if (nds.w != 0.0f) {   // zero = sky, or outside the frame (zero-filled by the tensor copy)
                    float common = svgf_depth_weight<FAST>(cnd.w, nds.w, 0.2f);
                    float nw = svgf_normal_weight<FAST>(cn, xyz(nds));
                    float sl = sv_luma<FAST>(xyz(t_di[k]));
                    float w = svgf_luma_weight<FAST>(scdl, sl, 1.0f) * common * nw;
                    sdi = sdi + f3(sl, sl * sl, 1.0f) * f3s(w);
                    float gl = sv_luma<FAST>(xyz(t_gi[k]));
                    float wg = svgf_luma_weight<FAST>(scgl, gl, 1.0f) * common * nw;
                    sgi = sgi + f3(gl, gl * gl, 1.0f) * f3s(wg);
                }
            }
        }
        { float m1 = sdi.x / sdi.z, m2 = sdi.y / sdi.z; di_var = fabs_(m2 - m1 * m1) * 4.0f; }
        { float m1 = sgi.x / sgi.z, m2 = sgi.y / sgi.z; gi_var = fabs_(m2 - m1 * m1) * 4.0f; }
    }
    di_var = rmax(di_var, 0.0f); gi_var = rmax(gi_var, 0.0f);
    cam.di_diff_stash[i] = f4(xyz(cdi), di_var);
    cam.gi_diff_stash[i] = f4(xyz(cgi), gi_var);
}

// ---- tile-staged K22: tensor maps + launcher --------------------------------------------------
// A float4 image plane as a 2-D tensor of 8-byte elements (2W x H; the widest element type a tensor map
// takes, so that a (TW+2·HL)-pixel box row stays under the 256-element box limit), row pitch W·16 B, no
// swizzle / interleave, zero fill outside the frame.  Maps are cached per (plane, frame size, box).
typedef CUresult (*TensorMapEncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                      const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static TensorMapEncodeFn tensor_map_encoder() {
    static TensorMapEncodeFn fn = [] {
        void* p = nullptr; cudaDriverEntryPointQueryResult q = cudaDriverEntryPointSymbolNotFound;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) p = nullptr;
        return (TensorMapEncodeFn)p;
    }();
    return fn;
}
static bool wavelet_tensor_map(const float4* plane, int w, int h, int bw, int bh, CUtensorMap* out) {
    typedef std::tuple<const void*, int, int, int, int> Key;
    static std::map<Key, CUtensorMap> cache; static std::mutex mu;
    std::lock_guard<std::mutex> lock(mu);
    Key key(plane, w, h, bw, bh);
    auto it = cache.find(key);
    if (it != cache.end()) { *out = it->second; return true; }
    TensorMapEncodeFn enc = tensor_map_encoder();
    if (!enc) {   // no driver entry point for tensor maps: the callers fall back to the gather kernels; say so once
        static bool warned = false;
        if (!warned) { warned = true; std::fprintf(stderr, "strolle_b200: cuTensorMapEncodeTiled is not available from this driver; the tile-staged SVGF kernels are off\n"); }
        return false;
    }
    cuuint64_t dims[2] = {(cuuint64_t)w * 2u, (cuuint64_t)h};
    cuuint64_t strides[1] = {(cuuint64_t)w * 16u};
    cuuint32_t box[2] = {(cuuint32_t)bw * 2u, (cuuint32_t)bh};
    cuuint32_t estr[2] = {1u, 1u};
    CUtensorMap tm;
    if (enc(&tm, CU_TENSOR_MAP_DATA_TYPE_UINT64, 2, const_cast<float4*>(plane), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS) return false;
    if (cache.size() > 4096) cache.clear();
    cache[key] = tm; *out = tm;
    return true;
}
template <bool FAST, int S, int J, int TW, int TH>
static bool wavelet_tiled_go(const CameraDev& c, const SceneDev& s, u32 frame, float strength, const float4* di_in, float4* di_out, const float4* gi_in, float4* gi_out,
                             float4* pair_out, u32* errors, cudaStream_t st) {
    typedef WaveletTile<S, J, TW, TH> T;
    if (T::BW * 2 > 256 || T::BH > 256) return false;
    CUtensorMap tn, td, tg;
    if (!wavelet_tensor_map(c.surface_nd, c.w, c.h, T::BW, T::BH, &tn) || !wavelet_tensor_map(di_in, c.w, c.h, T::BW, T::BH, &td) ||
        !wavelet_tensor_map(gi_in, c.w, c.h, T::BW, T::BH, &tg)) return false;
    auto kern = k_denoise_wavelet_tiled<FAST, S, J, TW, TH>;
    static bool attr_set[64] = {};   // per instantiation and device
    int dev = 0; cudaGetDevice(&dev); dev &= 63;
    if (!attr_set[dev]) { if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)T::SMEM) != cudaSuccess) { cudaGetLastError(); return false; } attr_set[dev] = true; }
    dim3 grid((c.w + TW - 1) / TW, (c.y1 - c.y0 + TH - 1) / TH);
    kern<<<grid, TW * TH, T::SMEM, st>>>(c, s, frame, strength, tn, td, tg, di_out, gi_out, pair_out, errors);
    return true;
}
template <bool FAST, int S, int J>
static bool wavelet_tiled_cfg(int cfg, const CameraDev& c, const SceneDev& s, u32 frame, float strength, const float4* di_in, float4* di_out, const float4* gi_in, float4* gi_out,
                              float4* pair_out, u32* errors, cudaStream_t st) {
    switch (cfg) {
    case 0: return wavelet_tiled_go<FAST, S, J, 32, 8>(c, s, frame, strength, di_in, di_out, gi_in, gi_out, pair_out, errors, st);
    case 1: return wavelet_tiled_go<FAST, S, J, 32, 16>(c, s, frame, strength, di_in, di_out, gi_in, gi_out, pair_out, errors, st);
    case 2: return wavelet_tiled_go<FAST, S, J, 64, 4>(c, s, frame, strength, di_in, di_out, gi_in, gi_out, pair_out, errors, st);
    case 3: return wavelet_tiled_go<FAST, S, J, 64, 8>(c, s, frame, strength, di_in, di_out, gi_in, gi_out, pair_out, errors, st);
    default: return false;
    }
}
// Returns false when the tile-staged kernel cannot be used for this launch (the caller then runs the gather kernel):
// the camera's screen is not the buffer size, no tensor-map encoder, or an unknown configuration.
bool launch_denoise_wavelet_tiled(const CameraDev& c, const SceneDev& s, u32 frame, u32 stride, float strength, const float4* di_in, float4* di_out, const float4* gi_in,
                                  float4* gi_out, float4* pair_out, bool fast, int cfg, u32* errors, cudaStream_t st) {
    if (c.curr.screen.x != (float)c.w || c.curr.screen.y != (float)c.h) return false;   // zero fill == Camera::contains only then
#define ST_WT(S_, J_) (fast ? wavelet_tiled_cfg<true, S_, J_>(cfg, c, s, frame, strength, di_in, di_out, gi_in, gi_out, pair_out, errors, st) \
                            : wavelet_tiled_cfg<false, S_, J_>(cfg, c, s, frame, strength, di_in, di_out, gi_in, gi_out, pair_out, errors, st))
    switch (stride) {
    case 1: return ST_WT(1, 0);
    case 2: return ST_WT(2, 0);
    case 4: return ST_WT(4, 0);
    case 8: return ST_WT(8, 1);
    case 16: return ST_WT(16, 3);
    default: return false;
    }
#undef ST_WT
}
template <bool FAST>
static bool variance_tiled_go(const CameraDev& c, const SceneDev& s, int cur, u32* errors, cudaStream_t st) {
    typedef VarianceTile<32, 8> T;
    CUtensorMap tn, td, tg;
    if (!wavelet_tensor_map(c.surface_nd, c.w, c.h, T::BW, T::BH, &tn) || !wavelet_tensor_map(c.di_diff_curr_colors, c.w, c.h, T::BW, T::BH, &td) ||
        !wavelet_tensor_map(c.gi_diff_curr_colors, c.w, c.h, T::BW, T::BH, &tg)) return false;
    auto kern = k_denoise_variance_tiled<FAST, 32, 8>;
    static bool attr_set[64] = {};
    int dev = 0; cudaGetDevice(&dev); dev &= 63;
    if (!attr_set[dev]) { if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)T::SMEM) != cudaSuccess) { cudaGetLastError(); return false; } attr_set[dev] = true; }
    dim3 grid((c.w + 31) / 32, (c.y1 - c.y0 + 7) / 8);
    kern<<<grid, 256, T::SMEM, st>>>(c, s, cur, tn, td, tg, errors);
    return true;
}
bool launch_denoise_variance_tiled(const CameraDev& c, const SceneDev& s, int cur, bool fast, u32* errors, cudaStream_t st) {
    if (c.curr.screen.x != (float)c.w || c.curr.screen.y != (float)c.h) return false;   // zero fill == Camera::contains only then
    return fast ? variance_tiled_go<true>(c, s, cur, errors, st) : variance_tiled_go<false>(c, s, cur, errors, st);
}
void launch_composition(const CameraDev& c, const SceneDev& s, int cur, u32 mode, const float4* di_diff, const float4* gi_diff, cudaStream_t st) { k_composition<<<grid_full(c), ST_BLOCK, 0, st>>>(c, s, cur, mode, di_diff, gi_diff); }
void launch_taa_resolve(const CameraDev& c, const SceneDev& s, int cur, u32 mode, const float4* di_diff, const float4* gi_diff, const float4* hist_in, float4* hist_out,
                        float4 jit, cudaStream_t st) {
    const dim3 grid((c.w + TAA_TW - 1) / TAA_TW, (c.h + TAA_TH - 1) / TAA_TH);
    k_taa_resolve<<<grid, TAA_TW * TAA_TH, 0, st>>>(c, s, cur, mode, di_diff, gi_diff, hist_in, hist_out, jit);
}
void launch_output_rgba8(const CameraDev& c, const SceneDev& s, uchar4* out, cudaStream_t st) { k_output_rgba8<<<grid_full(c), ST_BLOCK, 0, st>>>(c, s, out); }
void launch_exposure_histogram(const CameraDev& c, u32* state, ExposureDev p, int sms, cudaStream_t st) {
    const u32 n = (u32)c.w * (u32)c.h;
    const u32 ctas = std::max(1u, std::min((n + EXPO_THREADS - 1) / EXPO_THREADS, (u32)ST_EXPO_CTAS_PER_SM * (u32)sms));
    k_exposure_histogram<<<ctas, EXPO_THREADS, 0, st>>>(c.output, n, state, p);
#if ST_EXPO_METER_LAUNCH
    k_exposure_meter<<<1, kExposureBins, 0, st>>>(state, p);
#endif
}
void launch_output_display(const CameraDev& c, const SceneDev& s, int op, const u32* state, ExposureDev p, uchar4* out, cudaStream_t st) {
    switch (op) {
    case 1: k_output_display<1><<<grid_full(c), ST_BLOCK, 0, st>>>(c, s, out, state, p); break;
    case 2: k_output_display<2><<<grid_full(c), ST_BLOCK, 0, st>>>(c, s, out, state, p); break;
    case 3: k_output_display<3><<<grid_full(c), ST_BLOCK, 0, st>>>(c, s, out, state, p); break;
    default: k_output_display<4><<<grid_full(c), ST_BLOCK, 0, st>>>(c, s, out, state, p); break;
    }
}
static dim3 grid_of(int w, int h) { return dim3((w + TILE_W - 1) / TILE_W, (h + TILE_H - 1) / TILE_H); }
void launch_bloom_pyramid(const CameraDev& c, const BloomLevels& lv, const u32* state, ExposureDev p, int tm, BloomDev b, cudaStream_t st) {
    const int L = lv.levels;
    k_bloom_down0<<<dim3((lv.w[0] + BLOOM_TX - 1) / BLOOM_TX, (lv.h[0] + BLOOM_TY - 1) / BLOOM_TY), BLOOM_TX * BLOOM_TY, 0, st>>>(
        c.output, c.w, c.h, lv.down[0], lv.w[0], lv.h[0], state, p, tm, b);
    int tail = L;   // the first level of the one-CTA tail (L: none)
    for (int k = 1; k < L && ST_BLOOM_TAIL_TEXELS > 0; k++) if (lv.w[k] * lv.h[k] <= ST_BLOOM_TAIL_TEXELS) { tail = k; break; }
    for (int k = 1; k < tail; k++) k_bloom_down<<<grid_of(lv.w[k], lv.h[k]), ST_BLOCK, 0, st>>>(lv.down[k - 1], lv.w[k - 1], lv.h[k - 1], lv.down[k], lv.w[k], lv.h[k]);
    if (tail < L) {
#if ST_BLOOM_TAIL_KIND == 0
        k_bloom_tail<<<1, BLOOM_TAIL_THREADS, 0, st>>>(lv, tail, b.scatter);
#else
        // shared memory per CTA: the tail's down and up levels (for the cluster, each level's chunk); at most 4096 texels per level
        // keeps one CTA's copy under 180 KB
        size_t texels = 0;
        for (int k = tail; k < L; k++) texels += (size_t)(lv.w[k] * lv.h[k] + (ST_BLOOM_TAIL_KIND == 2 ? ST_BLOOM_CLUSTER - 1 : 0)) / (ST_BLOOM_TAIL_KIND == 2 ? ST_BLOOM_CLUSTER : 1) * (k + 1 < L ? 2 : 1);
        const int smem = (int)(16 * texels);
#if ST_BLOOM_TAIL_KIND == 1
        cudaFuncSetAttribute(k_bloom_tail_smem, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        k_bloom_tail_smem<<<1, BLOOM_TAIL_THREADS, smem, st>>>(lv, tail, b.scatter);
#else
        cudaFuncSetAttribute(k_bloom_tail_cluster, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        cudaLaunchConfig_t cfg = {};
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeClusterDimension; attr[0].val.clusterDim.x = ST_BLOOM_CLUSTER; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
        cfg.gridDim = dim3(ST_BLOOM_CLUSTER); cfg.blockDim = dim3(BLOOM_TAIL_THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = st; cfg.attrs = attr; cfg.numAttrs = 1;
        cudaLaunchKernelEx(&cfg, k_bloom_tail_cluster, lv, tail, b.scatter);
#endif
#endif
    }
    for (int k = std::min(tail, L - 1) - 1; k >= 0; k--)
        k_bloom_up<<<grid_of(lv.w[k], lv.h[k]), ST_BLOCK, 0, st>>>(lv.down[k], lv.up[k + 1], lv.w[k], lv.h[k], lv.w[k + 1], lv.h[k + 1], lv.up[k], b.scatter);
}
void launch_output_bloom(const CameraDev& c, const SceneDev& s, int op, const u32* state, ExposureDev p, BloomDev b, const float4* up0, int w0, int h0,
                         uchar4* out, cudaStream_t st) {
    switch (op) {
    case 0: k_output_bloom<0><<<grid_full(c), ST_BLOCK, 0, st>>>(c, s, out, state, p, b, up0, w0, h0); break;
    case 1: k_output_bloom<1><<<grid_full(c), ST_BLOCK, 0, st>>>(c, s, out, state, p, b, up0, w0, h0); break;
    case 2: k_output_bloom<2><<<grid_full(c), ST_BLOCK, 0, st>>>(c, s, out, state, p, b, up0, w0, h0); break;
    case 3: k_output_bloom<3><<<grid_full(c), ST_BLOCK, 0, st>>>(c, s, out, state, p, b, up0, w0, h0); break;
    default: k_output_bloom<4><<<grid_full(c), ST_BLOCK, 0, st>>>(c, s, out, state, p, b, up0, w0, h0); break;
    }
}
void launch_depth_of_field(const CameraDev& c, const DofDev& p, const DofBufs& b, cudaStream_t st) {
    const dim3 grid(b.tx, b.ty);
    k_dof_coc<<<grid, DOF_THREADS, 0, st>>>(c, p, b.words, b.tile_m);
    const int rmax = (int)ceilf(p.R);
    if (rmax > ST_DOF_STAGE_MAX_RADIUS) {
        k_dof_gather<false><<<grid, DOF_THREADS, 0, st>>>(c.output, c.w, c.h, p, b.words, b.tile_m, b.taps, b.frame);
        return;
    }
    const int S = kDofTile + 2 * rmax;   // the stage of the largest radius the frame can gather with
    static bool attr_set[64] = {};
    int dev = 0; cudaGetDevice(&dev); dev &= 63;
    if (!attr_set[dev]) {   // the largest stage this build launches: (16 + 2 ST_DOF_STAGE_MAX_RADIUS)^2 texels of 20 bytes
        const int most = (kDofTile + 2 * ST_DOF_STAGE_MAX_RADIUS) * (kDofTile + 2 * ST_DOF_STAGE_MAX_RADIUS) * 20;
        if (cudaFuncSetAttribute(k_dof_gather<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, most) != cudaSuccess) {
            // the device cannot hold the stage: the global-memory gather gives the same words
            cudaGetLastError();
            k_dof_gather<false><<<grid, DOF_THREADS, 0, st>>>(c.output, c.w, c.h, p, b.words, b.tile_m, b.taps, b.frame);
            return;
        }
        attr_set[dev] = true;
    }
    k_dof_gather<true><<<grid, DOF_THREADS, S * S * 20, st>>>(c.output, c.w, c.h, p, b.words, b.tile_m, b.taps, b.frame);
}
void launch_ref_tracing(const CameraDev& c, const SceneDev& s, u32 depth, bool nmap, const LensDev* lens, cudaStream_t st) {
    const LensDev lnone{};
    const LensDev& l = lens ? *lens : lnone;
#define ST_RT(N_, L_) k_ref_tracing<N_, L_><<<grid_full(c), ST_BLOCK, 0, st>>>(c, s, depth, l)
    if (lens) { if (nmap) ST_RT(true, true); else ST_RT(false, true); }
    else { if (nmap) ST_RT(true, false); else ST_RT(false, false); }
#undef ST_RT
}
void launch_ref_shading(const CameraDev& c, const SceneDev& s, u32 seed, u32 depth, const LightGridDev* lg, const TexFilterDev* tf, const EnvMapDev* em,
                        const LensDev* lens, cudaStream_t st) {
    const LightGridDev none{};
    const LightGridDev& g = lg ? *lg : none;
    const TexFilterDev tnone{};
    const TexFilterDev& t = tf ? *tf : tnone;
    const EnvMapDev enone{};
    const EnvMapDev& m = em ? *em : enone;
    const LensDev lnone{};
    const LensDev& l = lens ? *lens : lnone;
    // LENS only at depth 0, where the primary ray is formed
#define ST_RS(L_, T_, E_) do { if (lens && depth == 0u) k_ref_shading<L_, T_, E_, true><<<grid_full(c), ST_BLOCK, 0, st>>>(c, s, seed, depth, g, t, m, l); \
                               else k_ref_shading<L_, T_, E_, false><<<grid_full(c), ST_BLOCK, 0, st>>>(c, s, seed, depth, g, t, m, l); } while (0)
    if (em) {
        if (tf) { if (lg) ST_RS(true, true, true); else ST_RS(false, true, true); }
        else { if (lg) ST_RS(true, false, true); else ST_RS(false, false, true); }
    } else {
        if (tf) { if (lg) ST_RS(true, true, false); else ST_RS(false, true, false); }
        else { if (lg) ST_RS(true, false, false); else ST_RS(false, false, false); }
    }
#undef ST_RS
}
// ST_OPT_TEXTURE_FILTER: one launch per level (split into launches of at most 65535 images, the grid's y limit), `first[k]` ..
// `first[k + 1]` the jobs of level k + 1, `blocks[k]` their widest grid; returns the first launch error
cudaError_t launch_texture_mips(const MipJob* jobs, const u32* first, const u32* blocks, int levels, const uchar4* atlas, uchar4* pool, const float* srgb,
                                cudaStream_t st) {
    for (int k = 0; k < levels; k++) {
        if (!blocks[k]) continue;
        for (u32 j = first[k]; j < first[k + 1]; j += 65535u) {
            const u32 n = min(first[k + 1] - j, 65535u);
            k_texture_mips<<<dim3(blocks[k], n), 256, 0, st>>>(jobs + j, atlas, pool, srgb);
            const cudaError_t err = cudaGetLastError();
            if (err != cudaSuccess) return err;
        }
    }
    return cudaSuccess;
}
void launch_bvh_heatmap(const CameraDev& c, const SceneDev& s, cudaStream_t st) { k_bvh_heatmap<<<grid_full(c), ST_BLOCK, 0, st>>>(c, s); }
void launch_trace_stream_closest(const SceneDev& s, const float4* rays, long n, float4* out, cudaStream_t st) { k_trace_stream_closest<<<(unsigned)((n + ST_BLOCK - 1) / ST_BLOCK), ST_BLOCK, 0, st>>>(s, rays, n, out); }
void launch_trace_stream_any(const SceneDev& s, const float4* rays, long n, u32* out, cudaStream_t st) { k_trace_stream_any<<<(unsigned)((n + ST_BLOCK - 1) / ST_BLOCK), ST_BLOCK, 0, st>>>(s, rays, n, out); }
void launch_math(int op, const float* a, const float* b, float* out, long n, cudaStream_t st) {
    if (op == 7) k_math_log2<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(a, out, n);
    else if (op == 8 || op == 9) k_math_envm<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(op, a, b, out, n);
    else k_math<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(op, a, b, out, n);
}
// ST_OPT_ENVIRONMENT_MAP_SAMPLING (DESIGN.md §2 "Environment map sampling"): one warp per row i.  Texel (i, j)'s weight is the
// largest RGB channel over rows i-1..i+1 (clamped) and columns j-1..j+1 (wrapped), times the row's sin theta (cdf[i] on entry); the
// row's conditional CDF is the f32 running sum of its weights in column order.  Every lane adds the 32 weights of a chunk in order,
// so the sum is the sequential one.
__device__ __forceinline__ float envdist_max3(float4 t) { return fmaxf(fmaxf(t.x, t.y), t.z); }
__device__ __forceinline__ float envdist_scan32(float w, float* acc, u32 n) {   // the running sum at this lane, over lanes 0..n-1
    const u32 lane = threadIdx.x & 31u;
    float mine = 0.0f;
    for (u32 q = 0; q < n; q++) {
        const float x = __shfl_sync(0xffffffffu, w, q);
        *acc = xadd(*acc, x);
        if (lane == q) mine = *acc;
    }
    return mine;
}
__global__ void __launch_bounds__(256) k_envdist_rows(const float4* __restrict__ texels, u32 w, u32 h, float* __restrict__ cdf) {
    const u32 i = blockIdx.x * 8u + (threadIdx.x >> 5), lane = threadIdx.x & 31u;
    if (i >= h) return;
    const float sin_theta = cdf[i];
    const u32 r0 = i ? i - 1u : 0u, r2 = i + 1u < h ? i + 1u : h - 1u;
    float* row = cdf + h + (size_t)i * w;
    float acc = 0.0f;
    for (u32 base = 0; base < w; base += 32u) {
        const u32 j = base + lane;
        float wt = 0.0f;
        if (j < w) {
            const u32 jl = j ? j - 1u : w - 1u, jr = j + 1u < w ? j + 1u : 0u;
            float m = 0.0f;
            for (u32 r : {r0, i, r2}) {
                const float4* t = texels + (size_t)r * w;
                m = fmaxf(m, fmaxf(envdist_max3(__ldg(t + jl)), fmaxf(envdist_max3(__ldg(t + j)), envdist_max3(__ldg(t + jr)))));
            }
            wt = xmul(m, sin_theta);
        }
        const float c = envdist_scan32(wt, &acc, min(32u, w - base));
        if (j < w) row[j] = c;
    }
}
// The marginal CDF: the f32 running sum of the rows' last conditional values, in row order, by one warp.
__global__ void __launch_bounds__(32) k_envdist_marginal(u32 w, u32 h, float* __restrict__ cdf) {
    const u32 lane = threadIdx.x & 31u;
    float acc = 0.0f;
    for (u32 base = 0; base < h; base += 32u) {
        const u32 i = base + lane;
        const float r = i < h ? cdf[h + (size_t)i * w + w - 1u] : 0.0f;
        const float c = envdist_scan32(r, &acc, min(32u, h - base));
        if (i < h) cdf[i] = c;
    }
}
void launch_envdist_build(const float4* texels, uint32_t w, uint32_t h, float* cdf, cudaStream_t st) {
    k_envdist_rows<<<(h + 7u) / 8u, 256, 0, st>>>(texels, w, h, cdf);
    k_envdist_marginal<<<1, 32, 0, st>>>(w, h, cdf);
}
void launch_light_grid_build(const LightGridDev& lg, const GpuLight* lights, cudaStream_t st) {
    const u32 ncell = lg.dims[0] * lg.dims[1] * lg.dims[2];
    k_light_grid_build<<<(ncell + 1u + 3u) / 4u, 128, 0, st>>>(lg, lights, ncell, const_cast<u32*>(lg.counts), const_cast<u32*>(lg.lists));
}
void launch_material_derive(const GpuMaterial* mats, u32 n, u32* packed, cudaStream_t st) { if (n) k_material_derive<<<(n + 127) / 128, 128, 0, st>>>(mats, n, packed); }
void launch_srgb_lut(float* lut, cudaStream_t st) { k_srgb_lut<<<1, 256, 0, st>>>(lut); }
void launch_unpack_lut(float* lut, cudaStream_t st) { k_unpack_lut<<<1, 256, 0, st>>>(lut); }
// ---- strips, fused transport: sequence flags between ranks + the temporal pull -------------------------------------------
// Flags live in each rank's own memory, word [slot * ST_PEER_MAX_RANKS + source rank]; a rank raises its word in a peer's array to
// the frame's sequence number with a system-scope release store after the kernels that produced the rows have completed
// (stream order + fence), and a consumer spins on its local words with acquire loads.  One warp, lane r <-> rank r.
ST_DEV void st_release_sys(u32* p, u32 v) { asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
ST_DEV u32 ld_acquire_sys(const u32* p) { u32 v; asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
__global__ void __launch_bounds__(32) k_strip_signal(const __grid_constant__ StripSync s, int slot, u32 seq, u32 dst_mask, int* reset_need, int h) {
    __threadfence_system();
    int r = (int)threadIdx.x;
    if (r < s.n_ranks && r != s.rank && ((dst_mask >> r) & 1u) && s.peer_flags[r] != nullptr) st_release_sys(s.peer_flags[r] + slot * ST_PEER_MAX_RANKS + s.rank, seq);
    if (reset_need != nullptr && r == 0) { reset_need[0] = h; reset_need[1] = -1; }
}
__global__ void __launch_bounds__(32) k_strip_wait(const __grid_constant__ StripSync s, int slot, u32 seq, u32 src_mask) {
    int r = (int)threadIdx.x;
    if (r < s.n_ranks && r != s.rank && ((src_mask >> r) & 1u)) {
        const u32* f = s.my_flags + slot * ST_PEER_MAX_RANKS + r;
        long long t0 = clock64();
        while ((int)(ld_acquire_sys(f) - seq) < 0) {
            if (clock64() - t0 > 20000000000ll) {   // ~10 s: a peer died; do not hang the GPU.  errors[1] keeps the first wait that gave up
                atomicAdd(s.errors, 1u); atomicCAS(s.errors + 1, 0u, 0x80000000u | ((u32)slot << 16) | ((u32)r << 8) | (seq & 0xffu)); break;
            }
            __nanosleep(64);
        }
    }
    __threadfence_system();
}
// Temporal pull: rows [need_lo, own_y0) and [own_y1, need_hi] of last frame's outputs, read from their owners' arenas over NVLink
// (P2P loads).  The row range was measured on the device by this frame's G-buffer pass, so a static camera pulls nothing and
// any amount of motion is covered exactly.  blockIdx.y = buffer.
__global__ void __launch_bounds__(256) k_strip_pull(const __grid_constant__ StripPull p) {
    const int lo = max(0, min(p.need_rows[0], p.own_y0)), hi = min(p.h - 1, max(p.need_rows[1], p.own_y1 - 1));
    const StripPullItem it = p.items[blockIdx.y];
    // rows this rank already holds because it computes them itself (the extended G-buffer rows of the previous frame)
    const int have_lo = max(0, p.own_y0 - it.local_rows), have_hi = min(p.h, p.own_y1 + it.local_rows);
    const int up0 = lo, up1 = min(p.own_y0, have_lo), dn0 = max(p.own_y1, have_hi), dn1 = hi + 1;
    const int nup = max(0, up1 - up0), ndn = max(0, dn1 - dn0);
    const unsigned long long per_row = (unsigned long long)p.w * (unsigned long long)it.vec4_per_px;
    const unsigned long long total = (unsigned long long)(nup + ndn) * per_row;
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (unsigned long long)gridDim.x * blockDim.x) {
        int ri = (int)(i / per_row);
        unsigned long long col = i - (unsigned long long)ri * per_row;
        int row = ri < nup ? up0 + ri : dn0 + (ri - nup);
        int owner = 0;
        while (owner + 1 < p.n_ranks && row >= p.bounds[owner + 1]) owner++;
        size_t off = it.offset + ((size_t)row * per_row + col) * 16;
        *reinterpret_cast<uint4*>(p.arena[p.rank] + off) = *reinterpret_cast<const uint4*>(p.arena[owner] + off);
    }
    // statistics: rows of last frame this strip reached into, beyond its own (whatever part of them a buffer then had to fetch)
    if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) { int reach = max(0, p.own_y0 - lo) + max(0, hi + 1 - p.own_y1); if (reach > 0) atomicAdd(p.pulled_rows, (unsigned long long)reach); }
}
// a signal and a wait that follow each other on the stream, as one launch
__global__ void __launch_bounds__(32) k_strip_signal_wait(const __grid_constant__ StripSync s, int sig_slot, u32 seq, u32 dst_mask, int wait_slot, u32 wait_seq, u32 src_mask) {
    __threadfence_system();
    int r = (int)threadIdx.x;
    if (r < s.n_ranks && r != s.rank && ((dst_mask >> r) & 1u) && s.peer_flags[r] != nullptr) st_release_sys(s.peer_flags[r] + sig_slot * ST_PEER_MAX_RANKS + s.rank, seq);
    if (r < s.n_ranks && r != s.rank && ((src_mask >> r) & 1u)) {
        const u32* f = s.my_flags + wait_slot * ST_PEER_MAX_RANKS + r;
        long long t0 = clock64();
        while ((int)(ld_acquire_sys(f) - wait_seq) < 0) {
            if (clock64() - t0 > 20000000000ll) { atomicAdd(s.errors, 1u); break; }
            __nanosleep(64);
        }
    }
    __threadfence_system();
}
void launch_strip_signal_wait(const StripSync& s, int sig_slot, u32 seq, u32 dst_mask, int wait_slot, u32 wait_seq, u32 src_mask, cudaStream_t st) { k_strip_signal_wait<<<1, 32, 0, st>>>(s, sig_slot, seq, dst_mask, wait_slot, wait_seq, src_mask); }
void launch_strip_signal(const StripSync& s, int slot, u32 seq, u32 dst_mask, int* reset_need, int h, cudaStream_t st) { k_strip_signal<<<1, 32, 0, st>>>(s, slot, seq, dst_mask, reset_need, h); }
void launch_strip_wait(const StripSync& s, int slot, u32 seq, u32 src_mask, cudaStream_t st) { k_strip_wait<<<1, 32, 0, st>>>(s, slot, seq, src_mask); }
void launch_strip_pull(const StripPull& p, cudaStream_t st) { if (p.nitems > 0) k_strip_pull<<<dim3(48, (unsigned)p.nitems), 256, 0, st>>>(p); }

// ---- strips: push boundary rows into the neighbours' buffers, then barrier --------------------------------------
// One launch per exchange point.  blockIdx.y = segment (a run of rows of one buffer for one peer), blockIdx.x strides
// it with 16-byte stores that land in the peer's HBM through NVLink.  The last block to finish (completion counter)
// publishes `seq` in every peer's flag array after a system-scope fence and then spins until every peer has published
// the same `seq` here, so the next kernel on this stream sees all incoming rows.  Every exchange is a barrier over all
// ranks, which also orders a buffer's next overwrite after its last remote read.
__global__ void __launch_bounds__(256) k_peer_exchange(const __grid_constant__ PeerExchange x) {
    if (x.nseg > 0) {
        const PeerSegment& sg = x.seg[blockIdx.y];
        const uint4* __restrict__ src = sg.src; uint4* __restrict__ dst = sg.dst;
        for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < sg.n; i += (unsigned long long)gridDim.x * blockDim.x) dst[i] = src[i];
    }
    if (!x.signal) return;
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x != 0) return;
    unsigned total = gridDim.x * gridDim.y;
    if (atomicAdd(x.counter, 1u) != total - 1u) return;
    *x.counter = 0u;
    __threadfence_system();
    for (int r = 0; r < x.n_ranks; r++) if (r != x.rank) *(volatile u32*)x.peer_flags[r] = x.seq;
    long long t0 = clock64();
    for (int r = 0; r < x.n_ranks; r++) {
        if (r == x.rank) continue;
        const volatile u32* f = x.my_flags + r;
        while ((int)(*f - x.seq) < 0) {
            if (clock64() - t0 > 20000000000ll) { atomicAdd(x.errors, 1u); break; }   // ~10 s: a peer died; do not hang the GPU
            __nanosleep(100);
        }
    }
    __threadfence_system();
}
void launch_peer_exchange(const PeerExchange& x, cudaStream_t st) {
    unsigned ny = x.nseg > 0 ? (unsigned)x.nseg : 1u;
    unsigned nx = x.nseg > 0 ? std::max(4u, std::min(64u, 1184u / ny)) : 1u;
    k_peer_exchange<<<dim3(nx, ny), 256, 0, st>>>(x);
}
void launch_atm_transmittance(float4* out, cudaStream_t st) { k_atm_transmittance<<<dim3(2, 64), 128, 0, st>>>(out); }
void launch_atm_scattering(const float4* tl, float4* out, cudaStream_t st) { k_atm_scattering<<<32, 32, 0, st>>>(tl, out); }
void launch_atm_sky(const float4* tl, const float4* sl, float sun_altitude, float4* out, cudaStream_t st) { k_atm_sky<<<256, 256, 0, st>>>(tl, sl, sun_altitude, out); }
void launch_atm_sun_color(float4* out2, const GpuWorld& world, cudaStream_t st) { k_atm_sun_color<<<1, 1, 0, st>>>(out2, world); }

#endif   // ST_EXACT_ONLY

// Load every kernel of this translation unit's module now.  CUDA loads kernels lazily, at their first launch, and that load can
// synchronise the whole context; the strip transport lets one stream spin on a flag that a kernel launched later (by the same host
// thread, for another member of a device group) raises, so a load at that moment would stall the thread until the wait gives up.
// The module is found through one of its kernels; every function it holds is then loaded (cuFuncLoad, CUDA >= 12.4).
int preload_kernels() {
    static int states[64];   // per flavour (this function is compiled into st:: and stf::) and per device: every context holds its own copy of the module
    static bool init = false;
    if (!init) { for (int& v : states) v = -1; init = true; }
    int dev = 0; cudaGetDevice(&dev);
    int& state = states[dev & 63];
    if (state >= 0) return state;
    auto entry = [](const char* name) -> void* {
        void* p = nullptr; cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) return nullptr;
        return p;
    };
    typedef CUresult (*GetModule)(CUmodule*, CUfunction);
    typedef CUresult (*GetCount)(unsigned int*, CUmodule);
    typedef CUresult (*Enumerate)(CUfunction*, unsigned int, CUmodule);
    typedef CUresult (*Load)(CUfunction);
    GetModule get_module = (GetModule)entry("cuFuncGetModule"); GetCount get_count = (GetCount)entry("cuModuleGetFunctionCount");
    Enumerate enumerate = (Enumerate)entry("cuModuleEnumerateFunctions"); Load load = (Load)entry("cuFuncLoad");
    cudaGetLastError();
    if (!get_module || !get_count || !enumerate || !load) return state = 1;
    cudaFunction_t anchor = nullptr;
    if (cudaGetFuncBySymbol(&anchor, (const void*)k_di_sample_temporal<false>) != cudaSuccess) { cudaGetLastError(); return state = 2; }
    CUmodule mod = nullptr; unsigned int n = 0;
    if (get_module(&mod, (CUfunction)anchor) != CUDA_SUCCESS || get_count(&n, mod) != CUDA_SUCCESS || n == 0u) return state = 3;
    std::vector<CUfunction> fns(n);
    if (enumerate(fns.data(), n, mod) != CUDA_SUCCESS) return state = 4;
    for (CUfunction f : fns) if (load(f) != CUDA_SUCCESS) return state = 5;
    return state = 0;
}
}  // namespace ST_NS
