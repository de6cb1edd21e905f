// strolle_b200 — host-callable launchers for the kernels in kernels.cu.
#pragma once
#include <cuda_runtime.h>
#include "st_types.h"

namespace st {
typedef uint32_t u32;

// nmap: the NMAP instantiation (normal-mapped shading normal, ST_OPT_NORMAL_MAPS) of the kernels that shade a closest hit;
// tf (non-null): their TEXF instantiation (filtered material textures, ST_OPT_TEXTURE_FILTER); em (non-null): the ENVM instantiation
// of the kernels that evaluate the sky (K10, K13 and the fused K12 + K13, K2: the environment map of st_set_environment_map); K12, K13
// and the fused K12 + K13 run their ENV_SAMPLED instantiation when em->cdf is non-null (ST_OPT_ENVIRONMENT_MAP_SAMPLING)
void launch_prim_gbuffer(const CameraDev& c, const SceneDev& s, int cur, int with_reprojection, bool nmap, const TexFilterDev* tf, cudaStream_t st);
void launch_frame_reprojection(const CameraDev& c, const SceneDev& s, int cur, cudaStream_t st);
void launch_di_sampling(const CameraDev& c, const SceneDev& s, int cur, u32 seed, u32 frame, const LightGridDev* lg, cudaStream_t st);
void launch_di_temporal(const CameraDev& c, const SceneDev& s, int cur, u32 seed, cudaStream_t st);
void launch_di_spatial_pick(const CameraDev& c, const SceneDev& s, int cur, u32 seed, u32 frame, cudaStream_t st);
void launch_spatial_trace(const CameraDev& c, const SceneDev& s, const float4* d0, const float4* d1, float4* d2, cudaStream_t st);
void launch_di_spatial_sample(const CameraDev& c, const SceneDev& s, u32 seed, u32 frame, cudaStream_t st);
void launch_di_resolving(const CameraDev& c, const SceneDev& s, int cur, const EnvMapDev* em, cudaStream_t st);
void launch_gi_reprojection(const CameraDev& c, const SceneDev& s, int cur, cudaStream_t st);
void launch_gi_sampling_a(const CameraDev& c, const SceneDev& s, int cur, u32 seed, u32 frame, bool nmap, const TexFilterDev* tf, const EnvMapDev* em, cudaStream_t st);
void launch_gi_sampling_b(const CameraDev& c, const SceneDev& s, int cur, u32 seed, u32 frame, const LightGridDev* lg, const EnvMapDev* em, cudaStream_t st);
void launch_gi_temporal(const CameraDev& c, const SceneDev& s, int cur, u32 seed, u32 frame, int inline_reprojection, cudaStream_t st);
void launch_gi_spatial_pick(const CameraDev& c, const SceneDev& s, int cur, u32 seed, u32 frame, cudaStream_t st);
void launch_gi_spatial_sample(const CameraDev& c, const SceneDev& s, u32 seed, u32 frame, cudaStream_t st);
void launch_gi_preview(const CameraDev& c, const SceneDev& s, int cur, u32 seed, u32 nth, const float4* in, float4* out, int mirror_reach, cudaStream_t st);
void launch_gi_resolving(const CameraDev& c, const SceneDev& s, int cur, const float4* in, cudaStream_t st);
void launch_di_sample_temporal(const CameraDev& c, const SceneDev& s, int cur, u32 seed_sampling, u32 seed_temporal, u32 frame, const LightGridDev* lg, cudaStream_t st);
void launch_di_spatial_fused(const CameraDev& c, const SceneDev& s, int cur, u32 seed_pick, u32 seed_sample, u32 frame, cudaStream_t st);
void launch_gi_sampling_fused(const CameraDev& c, const SceneDev& s, int cur, u32 seed_a, u32 seed_b, u32 frame, bool nmap, const LightGridDev* lg, const TexFilterDev* tf,
                              const EnvMapDev* em, cudaStream_t st);
void launch_gi_spatial_fused(const CameraDev& c, const SceneDev& s, int cur, u32 seed_pick, u32 seed_sample, u32 frame, cudaStream_t st);
void launch_gi_preview_resolve(const CameraDev& c, const SceneDev& s, int cur, u32 seed, const float4* in, const float4* source, cudaStream_t st);
void launch_denoise_reproject(const CameraDev& c, const SceneDev& s, int cur, const float4* pc, const float4* pm, const float4* smp, float4* col, float4* mom, cudaStream_t st);
void launch_denoise_reproject_pair(const CameraDev& c, const SceneDev& s, int cur, cudaStream_t st);
void launch_denoise_variance(const CameraDev& c, const SceneDev& s, int cur, bool fast, cudaStream_t st);
void launch_denoise_wavelet(const CameraDev& c, const SceneDev& s, int cur, u32 frame, u32 stride, float strength, const float4* di_in, float4* di_out, const float4* gi_in, float4* gi_out, const float4* pair_in, float4* pair_out, bool fast, cudaStream_t st);
bool launch_denoise_wavelet_tiled(const CameraDev& c, const SceneDev& s, u32 frame, u32 stride, float strength, const float4* di_in, float4* di_out, const float4* gi_in, float4* gi_out, float4* pair_out, bool fast, int cfg, u32* errors, cudaStream_t st);
bool launch_denoise_variance_tiled(const CameraDev& c, const SceneDev& s, int cur, bool fast, u32* errors, cudaStream_t st);
void launch_composition(const CameraDev& c, const SceneDev& s, int cur, u32 mode, const float4* di_diff, const float4* gi_diff, cudaStream_t st);
// ST_OPT_TEMPORAL_AA: composes the frame (as launch_composition) into shared memory and resolves it against last frame's history
// (hist_in) into `output` and hist_out; jit = (J(f), J(f - 1)) in pixels, c.curr / c.prev the jittered cameras (strict build only)
void launch_taa_resolve(const CameraDev& c, const SceneDev& s, int cur, u32 mode, const float4* di_diff, const float4* gi_diff, const float4* hist_in, float4* hist_out,
                        float4 jit, cudaStream_t st);
void launch_output_rgba8(const CameraDev& c, const SceneDev& s, uchar4* out, cudaStream_t st);
// ST_OPT_TONEMAPPING / ST_OPT_AUTO_EXPOSURE (DESIGN.md §2 "Exposure and tonemapping"; strict build only).  The per-camera metering state,
// 32-bit words: {ev, target (f32 bits), counted, kept, frames}, the 256 bins of the last metered frame, the last-CTA ticket, then (at
// kExposureAccum) the 256 bins the next histogram accumulates into, zero between launches.
struct ExposureDev { float ev, compensation, ev_min, ev_max, low, high, speed_up, speed_down; };
enum { kExposureBins = 256, kExposureTicket = 5 + kExposureBins, kExposureAccum = 264, kExposureWords = kExposureAccum + kExposureBins };
// The log-luminance histogram of c.output (the whole frame) into state[kExposureAccum ..] over a grid sized from the device's `sms`
// multiprocessors; the last CTA to finish meters it, adapts the EV (state[0]) and zeroes the accumulator and the ticket for the next frame.
void launch_exposure_histogram(const CameraDev& c, u32* state, ExposureDev p, int sms, cudaStream_t st);
// The Rgba8 store of rows [c.y0, c.y1) through exposure 2^(compensation - ev) and the display transform `op` (1..4); ev = state[0]
// when `state` is non-null (auto exposure), p.ev otherwise
void launch_output_display(const CameraDev& c, const SceneDev& s, int op, const u32* state, ExposureDev p, uchar4* out, cudaStream_t st);
// ST_OPT_BLOOM (DESIGN.md §2 "Bloom"; strict build only).  The per-camera pyramid: kBloomHeaderWords 32-bit words {L, w_0, h_0, ..,
// w_7, h_7, 0, 0, 0} (zero past level L - 1), then float4 texels {r, g, b, 0}: the down levels 0 .. L - 1, then the up levels
// 0 .. L - 2 (up_{L-1} is down_{L-1}).  Level k is max(1, W >> (k + 1)) x max(1, H >> (k + 1)).
struct BloomDev { float intensity, scatter, threshold, softness; int levels, mode; };
enum { kBloomMaxLevels = 8, kBloomHeaderWords = 20 };
struct BloomLevels { float4* down[kBloomMaxLevels]; float4* up[kBloomMaxLevels]; int w[kBloomMaxLevels], h[kBloomMaxLevels]; int levels; };
// The levels of a W x H frame's pyramid of L levels at `base` (null: sizes only); returns the storage's size in bytes
inline size_t bloom_layout(int W, int H, int L, void* base, BloomLevels* lv) {
    float4* p = base ? (float4*)((char*)base + 4 * kBloomHeaderWords) : nullptr;
    size_t n = 0;
    lv->levels = L;
    for (int k = 0; k < kBloomMaxLevels; k++) {
        lv->w[k] = k < L ? ((W >> (k + 1)) > 1 ? (W >> (k + 1)) : 1) : 0;
        lv->h[k] = k < L ? ((H >> (k + 1)) > 1 ? (H >> (k + 1)) : 1) : 0;
        lv->down[k] = lv->up[k] = nullptr;
    }
    for (int k = 0; k < L; k++) { lv->down[k] = p ? p + n : nullptr; n += (size_t)lv->w[k] * lv->h[k]; }
    for (int k = 0; k + 1 < L; k++) { lv->up[k] = p ? p + n : nullptr; n += (size_t)lv->w[k] * lv->h[k]; }
    lv->up[L - 1] = lv->down[L - 1];
    return 4 * kBloomHeaderWords + 16 * n;
}
// The pyramid of c.output (the whole frame) through the input clamp, exposure (tm != 0: 2^(compensation - ev), ev = state[0] when
// `state` is non-null, p.ev otherwise), the prefilter and the down and up chains
void launch_bloom_pyramid(const CameraDev& c, const BloomLevels& lv, const u32* state, ExposureDev p, int tm, BloomDev b, cudaStream_t st);
// The Rgba8 store of rows [c.y0, c.y1) with the glow of up_0 composited: op 0 today's store, 1..4 exposed and tonemapped as
// launch_output_display
void launch_output_bloom(const CameraDev& c, const SceneDev& s, int op, const u32* state, ExposureDev p, BloomDev b, const float4* up0, int w0, int h0,
                         uchar4* out, cudaStream_t st);
// ST_OPT_DEPTH_OF_FIELD (DESIGN.md §2 "Depth of field"; strict build only).  16 x 16 pixel tiles; the gather's tap table holds, per
// radius rho = 1..kDofMaxRadius, kDofTaps integer offsets and their distances (dof_tap_table, engine.cu).  The per-camera buffer:
// the defocused frame (W x H float4), then the "depth_of_field" words {W, H, TX, TY, defocused, f, A, k, F, R, forward.xyz, 0, 0, 0}
// (kDofHeaderWords), the signed CoC radius r of every pixel and every tile's gather radius rho_t (u32), then every tile's max |r|
// (float) and the tap table; each section starts on a 256-byte boundary.
enum { kDofTile = 16, kDofMaxRadius = 32, kDofTaps = 81, kDofHeaderWords = 16 };
struct DofTap { short dx, dy; float d; };
struct DofDev {
    u32 head[kDofHeaderWords];   // the header words of the frame, as above
    int active;                  // 0: not defocused this frame (F <= f): every r is 0 and the frame is copied
    float k, F, R, fwd_x, fwd_y, fwd_z;
    int reach;                   // ceil(R / 16): the tiles a circle of radius R can reach
};
struct DofBufs { float4* frame; float* words; float* tile_m; const DofTap* taps; int tx, ty; size_t words_count; };
inline size_t dof_layout(int W, int H, void* base, DofBufs* b) {
    auto up = [](size_t n) { return (n + 255) / 256 * 256; };
    const size_t px = (size_t)W * H;
    b->tx = (W + kDofTile - 1) / kDofTile; b->ty = (H + kDofTile - 1) / kDofTile;
    const size_t tiles = (size_t)b->tx * b->ty;
    b->words_count = kDofHeaderWords + px + tiles;
    const size_t o_words = up(16 * px), o_m = o_words + up(4 * b->words_count), o_taps = o_m + up(4 * tiles);
    char* p = (char*)base;
    b->frame = p ? (float4*)p : nullptr; b->words = p ? (float*)(p + o_words) : nullptr;
    b->tile_m = p ? (float*)(p + o_m) : nullptr; b->taps = p ? (const DofTap*)(p + o_taps) : nullptr;
    return o_taps + sizeof(DofTap) * kDofMaxRadius * kDofTaps;
}
// The CoC of every pixel of c.surface_nd through c.curr's rays, each tile's max |r|, then the gather of c.output into b.frame
void launch_depth_of_field(const CameraDev& c, const DofDev& p, const DofBufs& b, cudaStream_t st);
// ST_OPT_DEPTH_OF_FIELD in Reference mode (DESIGN.md §2 "Depth of field"): the thin lens of K1 / K2's primary rays.  `seed` is the
// frame's lens dispatch seed; h = A / 2 the aperture radius; F the focal distance; right, up and fwd the camera's unit axes.
struct LensDev { u32 seed; float h, F, rx, ry, rz, ux, uy, uz, fx, fy, fz; };
// lens (non-null): the LENS instantiations, whose depth-0 ray is the thin-lens ray of `lens`
void launch_ref_tracing(const CameraDev& c, const SceneDev& s, u32 depth, bool nmap, const LensDev* lens, cudaStream_t st);
void launch_ref_shading(const CameraDev& c, const SceneDev& s, u32 seed, u32 depth, const LightGridDev* lg, const TexFilterDev* tf, const EnvMapDev* em,
                        const LensDev* lens, cudaStream_t st);
void launch_bvh_heatmap(const CameraDev& c, const SceneDev& s, cudaStream_t st);
void launch_trace_stream_closest(const SceneDev& s, const float4* rays, long n, float4* out, cudaStream_t st);
void launch_trace_stream_any(const SceneDev& s, const float4* rays, long n, u32* out, cudaStream_t st);
void launch_math(int op, const float* a, const float* b, float* out, long n, cudaStream_t st);
// ST_OPT_LIGHT_GRID: fills lg.counts / lg.lists (dims.x * dims.y * dims.z cells, then the outside list) from the device lights
void launch_light_grid_build(const LightGridDev& lg, const GpuLight* lights, cudaStream_t st);
// ST_OPT_ENVIRONMENT_MAP_SAMPLING: the distribution of `texels` (w x h) into `cdf` (h + w h floats, DESIGN.md §2 "Environment map
// sampling"); cdf[0 .. h) holds each row's sin theta on entry (k_envdist_rows reads it before k_envdist_marginal overwrites it)
void launch_envdist_build(const float4* texels, uint32_t w, uint32_t h, float* cdf, cudaStream_t st);
// ST_OPT_TEXTURE_FILTER: k_texture_mips for level k + 1 over jobs [first[k], first[k + 1]) with blocks[k] x 256 threads, k < levels,
// in launches of at most 65535 jobs; returns the first launch error
cudaError_t launch_texture_mips(const MipJob* jobs, const u32* first, const u32* blocks, int levels, const uchar4* atlas, uchar4* pool, const float* srgb, cudaStream_t st);
void launch_material_derive(const GpuMaterial* mats, u32 n, u32* packed, cudaStream_t st);
void launch_srgb_lut(float* lut, cudaStream_t st);
void launch_unpack_lut(float* lut, cudaStream_t st);
void launch_atm_transmittance(float4* out, cudaStream_t st);
void launch_atm_scattering(const float4* tl, float4* out, cudaStream_t st);
void launch_atm_sky(const float4* tl, const float4* sl, float sun_altitude, float4* out, cudaStream_t st);

// Halo rows over NVLink peer memory + device-side barrier (multi-GPU strips, SURVEY §8e)
#define ST_PEER_MAX_SEGMENTS 40
#define ST_PEER_MAX_RANKS 16
struct PeerSegment { const uint4* src; uint4* dst; unsigned long long n; };
struct PeerExchange {
    PeerSegment seg[ST_PEER_MAX_SEGMENTS]; int nseg;
    u32* peer_flags[ST_PEER_MAX_RANKS];   // slot [my rank] of every peer's flag array (mapped peer memory); null for self
    const u32* my_flags;                  // my flag array, slot [r] raised by rank r
    u32* counter; u32* errors;            // block completion counter (self-resetting), barrier time-out count
    int n_ranks, rank; u32 seq; int signal;
};
void launch_peer_exchange(const PeerExchange& x, cudaStream_t st);

// Fused strip transport (engine.cu render_strips_fused): sequence flags between ranks and the temporal pull
enum StripSlot { SLOT_FRAME_DONE = 0, SLOT_PULL_DONE = 1, SLOT_DI1 = 2, SLOT_GI1 = 3, SLOT_GI2 = 4, SLOT_GI3 = 5, SLOT_SVGF = 6, SLOT_GBUF = 7, SLOT_COUNT = 8 };
struct StripSync {
    const u32* my_flags;                  // this rank's flag words, [slot * ST_PEER_MAX_RANKS + source rank]
    u32* peer_flags[ST_PEER_MAX_RANKS];   // every other rank's flag array (mapped peer memory); null for self
    u32* errors;                          // wait time-outs
    int n_ranks, rank;
};
struct StripPullItem { size_t offset; int vec4_per_px; int local_rows; };   // arena byte offset of the buffer, float4 per pixel, rows beyond the strip this rank holds itself
struct StripPull {
    char* arena[ST_PEER_MAX_RANKS]; int bounds[ST_PEER_MAX_RANKS + 1];
    int n_ranks, rank, w, h, own_y0, own_y1;
    const int* need_rows; unsigned long long* pulled_rows;
    StripPullItem items[12]; int nitems;
};
int preload_kernels();   // 0 = every kernel of the strict build is loaded; > 0 = the driver cannot enumerate them (kernels then load at first launch)
void launch_strip_signal(const StripSync& s, int slot, u32 seq, u32 dst_mask, int* reset_need, int h, cudaStream_t st);
void launch_strip_wait(const StripSync& s, int slot, u32 seq, u32 src_mask, cudaStream_t st);
void launch_strip_signal_wait(const StripSync& s, int sig_slot, u32 seq, u32 dst_mask, int wait_slot, u32 wait_seq, u32 src_mask, cudaStream_t st);
void launch_strip_pull(const StripPull& p, cudaStream_t st);
void launch_atm_sun_color(float4* out2, const GpuWorld& world, cudaStream_t st);

// ST_OPT_BVH_REFIT (refit.cu).  One record per moved instance: its affine (x, y, z columns then translation), the transpose of the
// inverse's 3x3 (columns), the determinant's sign, its triangle range [b, e) in the triangle array, `first` = the thread index of
// its first triangle (prefix sum of the ranges), `tris` = its mesh's object-space st_mesh_triangles on the device.
struct BakeRecord { float xf[12]; float nt[9]; float sign; u32 b, e, first, pad; unsigned long long tris; };
void launch_bake_instances(const BakeRecord* recs, u32 nrec, u32 total, float4* triangles, cudaStream_t st);
// runs: {parent slot, first leaf entry, entry count, 0}; nodes: {ptr, parent slot} of every internal node but the root, grouped by level
// (deepest first, level l = [level_begin[l], level_begin[l + 1]))
void launch_refit(const uint4* runs, u32 nruns, const uint2* nodes, const u32* level_begin, int levels, const float4* triangles, float4* bvh, cudaStream_t st);

}  // namespace st

// The ReSTIR kernels K5-K19 built a second time with FMA contraction and SFU approximations (kernels.cu compiled with
// -DST_FAST=1, see st_math.cuh): same launch interface, selected by ST_OPT_SHADING_FAST_MATH.
namespace stf {
using st::CameraDev; using st::SceneDev; using st::LightGridDev; using st::TexFilterDev; using st::EnvMapDev; using st::u32;
int preload_kernels();   // the fast-shading build's kernels
void launch_di_sampling(const CameraDev& c, const SceneDev& s, int cur, u32 seed, u32 frame, const LightGridDev* lg, cudaStream_t st);
void launch_di_temporal(const CameraDev& c, const SceneDev& s, int cur, u32 seed, cudaStream_t st);
void launch_di_spatial_pick(const CameraDev& c, const SceneDev& s, int cur, u32 seed, u32 frame, cudaStream_t st);
void launch_spatial_trace(const CameraDev& c, const SceneDev& s, const float4* d0, const float4* d1, float4* d2, cudaStream_t st);
void launch_di_spatial_sample(const CameraDev& c, const SceneDev& s, u32 seed, u32 frame, cudaStream_t st);
void launch_di_resolving(const CameraDev& c, const SceneDev& s, int cur, const EnvMapDev* em, cudaStream_t st);
void launch_gi_reprojection(const CameraDev& c, const SceneDev& s, int cur, cudaStream_t st);
void launch_gi_sampling_a(const CameraDev& c, const SceneDev& s, int cur, u32 seed, u32 frame, bool nmap, const TexFilterDev* tf, const EnvMapDev* em, cudaStream_t st);
void launch_gi_sampling_b(const CameraDev& c, const SceneDev& s, int cur, u32 seed, u32 frame, const LightGridDev* lg, const EnvMapDev* em, cudaStream_t st);
void launch_gi_temporal(const CameraDev& c, const SceneDev& s, int cur, u32 seed, u32 frame, int inline_reprojection, cudaStream_t st);
void launch_gi_spatial_pick(const CameraDev& c, const SceneDev& s, int cur, u32 seed, u32 frame, cudaStream_t st);
void launch_gi_spatial_sample(const CameraDev& c, const SceneDev& s, u32 seed, u32 frame, cudaStream_t st);
void launch_gi_preview(const CameraDev& c, const SceneDev& s, int cur, u32 seed, u32 nth, const float4* in, float4* out, int mirror_reach, cudaStream_t st);
void launch_gi_resolving(const CameraDev& c, const SceneDev& s, int cur, const float4* in, cudaStream_t st);
void launch_di_sample_temporal(const CameraDev& c, const SceneDev& s, int cur, u32 seed_sampling, u32 seed_temporal, u32 frame, const LightGridDev* lg, cudaStream_t st);
void launch_di_spatial_fused(const CameraDev& c, const SceneDev& s, int cur, u32 seed_pick, u32 seed_sample, u32 frame, cudaStream_t st);
void launch_gi_sampling_fused(const CameraDev& c, const SceneDev& s, int cur, u32 seed_a, u32 seed_b, u32 frame, bool nmap, const LightGridDev* lg, const TexFilterDev* tf,
                              const EnvMapDev* em, cudaStream_t st);
void launch_gi_spatial_fused(const CameraDev& c, const SceneDev& s, int cur, u32 seed_pick, u32 seed_sample, u32 frame, cudaStream_t st);
void launch_gi_preview_resolve(const CameraDev& c, const SceneDev& s, int cur, u32 seed, const float4* in, const float4* source, cudaStream_t st);
void launch_math_shading(int op, const float* a, const float* b, float* out, long n, cudaStream_t st);   // test hook: this build's sin/cos/exp/pow/sqrt/div
}  // namespace stf
