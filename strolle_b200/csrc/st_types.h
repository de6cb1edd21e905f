// strolle_b200 — POD layouts shared by the host engine and the CUDA kernels.
// Wire layouts are byte-identical to strolle-gpu's #[repr(C)] structs
// (SURVEY.md Appendix A; reference files cited per struct).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace st {

struct GpuMaterial {   // strolle-gpu/src/material.rs:7-21, 112 B
    float4 base_color, base_color_texture, emissive, emissive_texture;
    float roughness, metallic, reflectance, ior;
    float4 metallic_roughness_texture, normal_map_texture;
};
struct GpuLight {      // strolle-gpu/src/light.rs:13-42, 112 B
    float4 d0, d1, d2, d3, prev_d0, prev_d1, prev_d2;
};
struct GpuWorld {      // strolle-gpu/src/world.rs:6-13
    uint32_t light_count; float sun_azimuth, sun_altitude; uint32_t pad;
};
struct GpuCamera {     // strolle-gpu/src/camera.rs:8-16, 160 B
    float4 projection_view[4], ndc_to_world[4], origin, screen;
};
static_assert(sizeof(GpuMaterial) == 112, "material layout");
static_assert(sizeof(GpuLight) == 112, "light layout");
static_assert(sizeof(GpuCamera) == 160, "camera layout");

static const uint32_t kAtlasSize = 8192;   // strolle/src/images.rs:29-30

// Scene-wide device pointers (replicated on every GPU).
struct SceneDev {
    const float4* triangles;   // 9 float4 per triangle (strolle-gpu/src/triangle.rs:8-21)
    const float4* bvh;         // strolle/src/bvh/serializer.rs:53-104
    uint32_t bvh_len;          // float4 count of `bvh`; 0 = no primitive alive (empty stream, serializer.rs:20-110): every ray misses
    const GpuMaterial* materials;
    const GpuLight* lights;
    const uchar4* blue_noise;  // 256x256 RGBA8
    const float4* transmittance_lut;   // 256x64, values rounded to f16
    const float4* scattering_lut;      // 32x32
    const float4* sky_lut;             // 256x256
    GpuWorld world;
    const uint32_t* tri_instance;      // per triangle: instance slot
    const float4* instance_xforms;     // per instance 6 float4: curr_xform_inv d0..d2, prev_xform d0..d2 (strolle-gpu/src/passes.rs:54-77)
    const uchar4* atlas;               // kAtlasSize^2 RGBA8 (Rgba8UnormSrgb), null until an image is inserted (strolle/src/images.rs:29-43)
    const float* srgb_lut;             // 256-entry sRGB -> linear table
    const uint32_t* material_packed;   // derived per material: byte-packed gamma-2.2 base colour (GBufferEntry::pack d1.w)
    const float* unpack_lut;           // derived: [0..255] pow(b/255, 2.2), [256..511] pow(b/63, 2.2) (GBufferEntry::unpack)
    unsigned long long* ray_counter;   // optional: counts executed Ray::trace / Ray::intersect calls (Mrays/s)
};

// ST_OPT_LIGHT_GRID (DESIGN.md §2 "Light grid"): the per-cell candidate lists of the light slots that can reach the cell.  Built on
// the device at st_tick (k_light_grid_build); passed by value to the LGRID instantiations of the candidate-sampling kernels only.
static const uint32_t kLightGridK = 64;                   // list capacity per cell
static const uint32_t kLightGridOverflow = 0xffffffffu;   // a count that marks an overflowing list: the cell samples every slot
struct LightGridDev {
    float lo[3];         // grid box minimum: the AABB of the cullable lights' spheres
    float cell[3];       // cell size per axis (extent / dims)
    float inv_cell[3];   // dims / extent: point -> cell index
    float band[3];       // in cells: points outside the box by less than this clamp to the edge cell instead of taking the outside list
    float margin[3];     // world units each cell box is grown by before the reach test
    uint32_t dims[3];
    uint32_t light_count;            // the slots the lists were built over
    const uint32_t* counts;          // dims.x * dims.y * dims.z cells + 1 (the outside list last); kLightGridOverflow = every slot
    const uint32_t* lists;           // kLightGridK slots per cell, the outside list last
};

// ST_OPT_TEXTURE_FILTER (DESIGN.md §2 "Texture filtering"): levels 1.. of every live image's mip chain, and per material and colour
// slot (base colour, emissive, metallic-roughness) {texel offset of the image's level 1 in `pool`, level count}: 0 = no texture, 1 =
// level 0 only (a 1x1 image, or a stale rect).  Built on the device at st_tick (k_texture_mips); passed by value to the TEXF
// instantiations of the hit-shading kernels only.
struct TexFilterDev {
    const uchar4* pool;     // RGBA8 texels: per image, level after level, each row-major
    const uint2* table;     // 3 entries per material
};
// One image of one k_texture_mips launch: level k+1 (dst_w x dst_h at `dst` in the pool) from level k (src_w x src_h, rows `src_stride`
// texels apart from `src`, in the atlas for k = 0, else in the pool)
struct MipJob { uint32_t src, src_stride, src_w, src_h, dst, dst_w, dst_h, from_atlas; };

// st_set_environment_map (DESIGN.md §2 "Environment map"): an equirectangular map of linear RGB in place of the procedural sky.
// Uploaded by st_set_environment_map, taken at st_tick; passed by value to the ENVM instantiations of the sky-evaluating kernels only.
struct EnvMapDev {
    const float4* texels;   // w x h, row-major, row 0 the zenith; alpha unused
    uint32_t w, h;
    float intensity;        // radiance scale
    float rotation;         // radians in [0, 2 pi), added to the azimuth
    // ST_OPT_ENVIRONMENT_MAP_SAMPLING (DESIGN.md §2 "Environment map sampling"): the marginal CDF (h floats) followed by the h
    // conditional CDFs (w floats each), and the marginal's last value; cdf is null (and the sampled instantiations do not run)
    // while the option is off or the map has no distribution
    const float* cdf;
    float total;
};
// The three instantiations of the GI sampling kernels (K12, K13 and both fused) by what their sky is
enum EnvMode { ENV_NONE = 0, ENV_MAP = 1, ENV_SAMPLED = 2 };

// Per-camera device buffers: the logical buffers of
// strolle/src/camera_controller/buffers.rs:53-339 as linear row-major float4
// arrays indexed by full-frame coordinates (each GPU of a strip-partitioned run
// holds full-frame arrays, computes rows [y0, y1) and receives halo rows).
struct CameraDev {
    GpuCamera curr, prev;
    int w, h;            // full-frame size (Camera::screen)
    int y0, y1;          // rows this device computes (row strip of a multi-GPU run), [y0, y1)
    float4* prim_gbuffer_d0[2]; float4* prim_gbuffer_d1[2]; float4* prim_surface_map[2];
    float4* reprojection_map; float4* velocity_map;
    float4* di_reservoirs[3];
    float4* di_diff_samples; float4* di_diff_prev_colors; float4* di_diff_curr_colors; float4* di_diff_moments[2]; float4* di_diff_stash; float4* di_spec_samples;
    float4* gi_d0; float4* gi_d1; float4* gi_d2; float4* gi_reservoirs[4];
    float4* gi_diff_samples; float4* gi_diff_prev_colors; float4* gi_diff_curr_colors; float4* gi_diff_moments[2]; float4* gi_diff_stash; float4* gi_spec_samples;
    float4* ref_hits; float4* ref_rays; float4* ref_colors;
    float4* prim_triangle_ids;
    float4* surface_nd;          // derived: (decoded surface normal.xyz, depth) of the current frame, written with the G-buffer
    float4* output;
    // Row-strip partition, fused transport (engine.cu render_strips_fused): the kernels that produce a buffer a neighbouring
    // strip gathers from (K6 di[1], K14 gi[1], K17 gi[2], K18#1 gi[3], K20 colours + moments) store the rows within reach of
    // the strip's edges a second time, straight into the neighbour's copy of the buffer over NVLink.  Arenas have the same
    // layout on every rank, so the remote address is the local one plus a constant byte offset.  0 = no neighbour there.
    long long mirror_up, mirror_dn;
    int gi_mirror_reach;         // rows of gi_reservoirs[1] / [2] the GI kernels mirror themselves (ST_REACH_SPATIAL), or 0 when those rows travel by copy engine after the kernel
    int di_mirror_reach;         // the same for di_reservoirs[1] (K6)
    int own_y0, own_y1;          // the rows this rank owns (mirror decisions); [y0, y1) may be wider when a pass recomputes halo rows
    int* need_rows;              // device: {min, max} previous-frame row the reprojection of the owned rows reaches (K0 -> temporal pull); null = off
};

// Kernel ids (also the explicit-seed dispatch ids and the timing slots).
enum PassId {
    P_PRIM_GBUFFER = 0, P_DI_SAMPLING = 1, P_DI_TEMPORAL = 2, P_DI_SPATIAL_PICK = 3, P_DI_SPATIAL_TRACE = 4, P_DI_SPATIAL_SAMPLE = 5,
    P_DI_RESOLVING = 6, P_GI_REPROJECTION = 7, P_GI_SAMPLING_A = 8, P_GI_SAMPLING_B = 9, P_GI_TEMPORAL = 10, P_GI_SPATIAL_PICK = 11,
    P_GI_SPATIAL_TRACE = 12, P_GI_SPATIAL_SAMPLE = 13, P_GI_PREVIEW = 14, P_GI_RESOLVING = 15, P_FRAME_REPROJECTION = 16,
    P_DENOISE_REPROJECT = 17, P_DENOISE_VARIANCE = 18, P_DENOISE_WAVELET = 19, P_COMPOSITION = 20, P_REF_TRACING = 21,
    P_REF_SHADING = 22, P_BVH_HEATMAP = 23, P_ATMOSPHERE = 24, P_TRACE_STREAM = 25, P_HALO_EXCHANGE = 26, P_COUNT = 27,
    P_REF_SHADING_SEED = 32
};

}  // namespace st
