/* strolle_b200 — C ABI of the H100-native Strolle hot path.
 *
 * Drop-in boundary for the per-pixel GI path of Patryk27/strolle: the functions
 * below are what a Rust `extern "C"` shim behind `strolle::Engine<P>` binds in
 * place of the wgpu compute dispatches (CameraComputePass::run,
 * strolle/src/camera_controller/pass.rs:33-63) and buffer flushes
 * (strolle/src/buffers/mapped_storage_buffer.rs:108-140).  Each entry point
 * cites the reference method it replaces.  Plain pointers and sizes only; no
 * torch / CUDA types.  See INTEGRATION.md for the reference-side binding.
 *
 * Conventions: every function returns ST_OK (0) or a negative error code and
 * never aborts across the ABI; st_last_error() gives the message (the
 * reference panics instead, e.g. strolle/src/triangles.rs:44-53).  Handles are
 * caller-chosen opaque u64 (the reference's Params associated types,
 * strolle/src/lib.rs:402-409).  Mutating calls are externally synchronised
 * (single writer), like `ResMut<Engine>` in bevy-strolle.
 */
#ifndef STROLLE_B200_H
#define STROLLE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct st_engine st_engine;
typedef uint64_t st_handle;
typedef int32_t st_camera_handle;

enum { ST_OK = 0, ST_ERR_CUDA = -1, ST_ERR_INVALID = -2, ST_ERR_NOT_FOUND = -3, ST_ERR_LIMIT = -4 };

/* strolle::MeshTriangle (strolle/src/mesh_triangle.rs:7-12), object space */
typedef struct st_mesh_triangle {
    float positions[3][3];
    float normals[3][3];
    float uvs[3][2];
    float tangents[3][4];
} st_mesh_triangle;

/* strolle::Material (strolle/src/material.rs:8-23); textures are a later row (SURVEY §8f-3) */
typedef struct st_material {
    float base_color[4];
    float emissive[4];
    float perceptual_roughness;
    float metallic;
    float reflectance;
    float ior;
    int32_t alpha_blend; /* AlphaMode::Blend != 0 (strolle/src/material.rs:76-91) */
} st_material;

/* strolle::Light::{Point,Spot} (strolle/src/light.rs:6-22) */
enum { ST_LIGHT_POINT = 1, ST_LIGHT_SPOT = 2 };
typedef struct st_light {
    int32_t kind;
    float position[3];
    float radius;
    float color[3];
    float range;
    float direction[3]; /* spot only */
    float angle;        /* spot only */
} st_light;

/* strolle::CameraMode (strolle/src/camera.rs:83-105) */
enum {
    ST_MODE_IMAGE = 0, ST_MODE_DI_DIFFUSE = 1, ST_MODE_DI_SPECULAR = 2, ST_MODE_GI_DIFFUSE = 3,
    ST_MODE_GI_SPECULAR = 4, ST_MODE_BVH_HEATMAP = 5, ST_MODE_REFERENCE = 6
};
/* strolle::Camera (strolle/src/camera.rs:8-14); matrices column-major like glam::Mat4 */
typedef struct st_camera {
    int32_t mode;
    int32_t denoise;   /* CameraMode::*{denoise} */
    int32_t ref_depth; /* CameraMode::Reference{depth} */
    uint32_t width, height; /* CameraViewport::size */
    float transform[16];
    float projection[16];
} st_camera;

/* Output pixel formats for st_render_camera (the reference composes into the caller's
 * TextureView of CameraViewport::format, strolle/src/camera.rs:170-185). */
enum { ST_FORMAT_RGBA32F = 0, ST_FORMAT_RGBA8_SRGB = 1 };

const char* st_last_error(void);

/* Engine::new (strolle/src/lib.rs:132-158).  `device` = CUDA ordinal. */
int st_engine_create(int device, st_engine** out);
void st_engine_destroy(st_engine* e);

/* Engine::insert_mesh / remove_mesh (lib.rs:161-171) */
int st_insert_mesh(st_engine* e, st_handle mesh, const st_mesh_triangle* triangles, size_t count);
int st_remove_mesh(st_engine* e, st_handle mesh);
/* Engine::insert_material / has_material / remove_material (lib.rs:174-195) */
int st_insert_material(st_engine* e, st_handle material, const st_material* m);
int st_has_material(st_engine* e, st_handle material);
int st_remove_material(st_engine* e, st_handle material);
/* Engine::insert_image / remove_image (lib.rs:198-214), ImageData::Raw only: tightly packed RGBA8 pixels in
 * the atlas format Rgba8UnormSrgb (strolle/src/images.rs:38-43).  ST_ERR_LIMIT when the 8192^2 atlas is full
 * (the reference warns and drops the image, images.rs:71-79). */
int st_insert_image(st_engine* e, st_handle image, const uint8_t* rgba8, uint32_t width, uint32_t height);
int st_remove_image(st_engine* e, st_handle image);
/* The Option<ImageHandle> fields of strolle::Material (strolle/src/material.rs:13-22); bit i of `mask` = texture i set
 * (0 base_color, 1 emissive, 2 metallic_roughness, 3 normal_map).  The normal map is ignored, as in the reference, unless
 * ST_OPT_NORMAL_MAPS is on; it is then decoded linearly (byte / 255), the other three with the sRGB curve. */
typedef struct st_material_textures { st_handle base_color, emissive, metallic_roughness, normal_map; uint32_t mask; } st_material_textures;
int st_set_material_textures(st_engine* e, st_handle material, const st_material_textures* textures);
/* Engine::insert_instance / remove_instance (lib.rs:217-229); affine = glam::Affine3A as
 * matrix3 columns x,y,z then translation (12 floats) */
int st_insert_instance(st_engine* e, st_handle instance, st_handle mesh, st_handle material, const float affine[12]);
int st_remove_instance(st_engine* e, st_handle instance);
/* Engine::insert_light / remove_light (lib.rs:232-239) */
int st_insert_light(st_engine* e, st_handle light, const st_light* l);
int st_remove_light(st_engine* e, st_handle light);
/* Engine::update_sun (lib.rs:242-245) */
int st_update_sun(st_engine* e, float azimuth, float altitude);
/* An equirectangular environment map in place of the procedural sky (default: none, the reference's atmosphere).  `rgba32f` holds
 * width x height texels of linear RGB (4 floats each, alpha ignored), row-major, row 0 the zenith; NULL clears the map (the procedural
 * sky comes back and the device copy is freed at the next st_tick).  The map's radiance along a direction d is the bilinear blend at
 * u = (atan2(d.x, -d.z) + rotation) / 2 pi + 0.5, v = acos(d.y) / pi (columns wrapped, rows clamped), times `intensity`: with
 * rotation 0 the centre column is seen looking down -Z, u = 0.75 looking down +X.  It replaces the sky at every site that evaluates it
 * (sky pixels, GI bounces that miss, the GI bounce's sky draw, Reference mode's miss) without the procedural sky's x20 exposure; the
 * GI sky draw keeps its probability of 0.25 whatever the sun's altitude.  The sun light still follows st_update_sun: to light a scene
 * from the map alone, put the sun below the horizon (altitude < 0: its colour is then 0).  ST_ERR_INVALID, and no change, when a side
 * is outside 1..16384, an RGB value is negative or not finite, `intensity` is negative or not finite, or `rotation` is not finite.
 * `rotation` is reduced into [0, 2 pi) in double, then rounded to f32.  Takes effect at the next st_tick, which uploads the texels;
 * ST_STAT_ENVIRONMENT_MAP_LAUNCHES counts the launches that evaluate it (DESIGN.md §2 "Environment map"). */
int st_set_environment_map(st_engine* e, const float* rgba32f, uint32_t width, uint32_t height, float intensity, float rotation);
/* The exposure of the tonemapped Rgba8 store (ST_OPT_TONEMAPPING, ST_OPT_AUTO_EXPOSURE), in stops: the stored value is scene value x
 * 2^(compensation - ev).  `ev`: the manual exposure; `compensation`: added in both modes; `ev_min` <= `ev_max`: the clamp on the
 * metered EV; `low` < `high` in [0, 1]: the metered fraction of the counted pixels (the darkest `low` and the brightest 1 - `high` are
 * dropped); `speed_up`, `speed_down` >= 0: the largest EV change per frame, up and down.  Every field must be finite. */
typedef struct st_exposure { float ev, compensation, ev_min, ev_max, low, high, speed_up, speed_down; } st_exposure;
/* NULL restores the defaults {0, 0, -8, 8, 0.1, 0.9, 0.05, 1/60}.  The whole call is validated first: ST_ERR_INVALID, and no change,
 * when a field is out of range.  Takes effect at the next st_tick. */
int st_set_exposure(st_engine* e, const st_exposure* exposure);
/* The glow of ST_OPT_BLOOM (DESIGN.md §2 "Bloom").  `intensity`: the glow's share of the stored value, in [0, 1] with `mode` 0
 * (energy-conserving: (1 - intensity) x + intensity B) or >= 0 with `mode` 1 (additive: x + intensity B); `scatter` in [0, 1]: how far
 * the glow spreads (level k of the pyramid weighs (1 - scatter) scatter^k, the last level scatter^(L-1)); `threshold` >= 0: the exposed
 * brightness max(r, g, b) where the glow starts (0: every pixel glows), with a soft knee of width threshold x `softness`, `softness` in
 * [0, 1]; `levels` in 1..8: the pyramid's depth L, level 0 at half resolution.  Every float field must be finite. */
typedef struct st_bloom { float intensity, scatter, threshold, softness; int32_t levels, mode; } st_bloom;
/* NULL restores the defaults {0.15, 0.7, 0, 0, 7, 0}.  The whole call is validated first: ST_ERR_INVALID, and no change, when a field
 * is out of range.  Takes effect at the next st_tick. */
int st_set_bloom(st_engine* e, const st_bloom* bloom);
/* The thin lens of ST_OPT_DEPTH_OF_FIELD (DESIGN.md §2 "Depth of field").  `focal_distance` (> 0, scene units): the view depth in
 * focus; `aperture_f_stops` (> 0): the f-number N; `sensor_height` (> 0, scene units): the sensor's height, which with the
 * projection's vertical field of view gives the focal length f = sensor_height P11 / 2 (P11 = projection[5]); `max_radius` in [1, 32]:
 * the largest radius of the circle of confusion, in output pixels.  Every field must be finite. */
typedef struct st_depth_of_field { float focal_distance, aperture_f_stops, sensor_height, max_radius; } st_depth_of_field;
/* NULL restores the defaults {10, 1, 0.01866, 16} (focus 10 units away at f/1 on a Super 35 sensor, 18.66 mm in metres, as Bevy's
 * DepthOfField uses).  The whole call is validated first: ST_ERR_INVALID, and no change, when a field is out of range.  Takes effect
 * at the next st_tick. */
int st_set_depth_of_field(st_engine* e, const st_depth_of_field* dof);

/* Engine::create_camera / update_camera / delete_camera (lib.rs:252-294) */
int st_create_camera(st_engine* e, const st_camera* camera, st_camera_handle* out);
int st_update_camera(st_engine* e, st_camera_handle camera, const st_camera* desc);
int st_delete_camera(st_engine* e, st_camera_handle camera);

/* Engine::tick (lib.rs:301-395): bakes dirty instances, rebuilds + uploads the BVH, lights,
 * materials, world; must precede st_render_camera each frame. */
int st_tick(st_engine* e);

/* Engine::render_camera (lib.rs:279-286 -> CameraController::render,
 * strolle/src/camera_controller.rs:87-174): runs the frame's pass schedule on the engine's
 * stream.  If `host_out` is non-NULL the composed frame (width*height pixels of `format`) is
 * copied to it and the call returns when the copy is done; with NULL the call only enqueues
 * (use st_synchronize). */
int st_render_camera(st_engine* e, st_camera_handle camera, void* host_out, int format);
/* Converts the camera's composed frame to `format` and copies it to host memory (what
 * st_render_camera does when host_out != NULL), without re-running the passes. */
int st_copy_output(st_engine* e, st_camera_handle camera, void* host_out, int format);
int st_synchronize(st_engine* e);

/* ---- hooks that the reference does not have (SURVEY §8b) -------------------------------- */
/* Explicit per-dispatch seeds: seed(frame f, dispatch k) = pcg(base ^ (f*64 + k)); the reference
 * draws rand::thread_rng() per dispatch (camera_controller.rs:189-194) and is not reproducible. */
int st_set_seed_base(st_engine* e, uint32_t base);
/* 256x256 RGBA8 blue-noise tile (strolle/src/noise.rs:30-66 embeds a PNG; here the host passes bytes) */
int st_set_blue_noise(st_engine* e, const uint8_t* rgba8_256x256);
/* Copies a per-camera buffer (names = fields of CameraBuffers, strolle/src/camera_controller/
 * buffers.rs:9-51; double-buffered ones take _a/_b) to host.  Returns #floats available via
 * *count; copies min(cap, count). */
int st_read_buffer(st_engine* e, st_camera_handle camera, const char* name, float* dst, size_t cap_floats, size_t* count);
/* Scene buffers as uploaded: "triangles", "bvh", "materials", "lights", "world", "transmittance_lut",
 * "scattering_lut", "sky_lut"; and, while ST_OPT_LIGHT_GRID is on and a tick has built it, "light_grid" as 32-bit words: a 21-word
 * header {dims x, y, z, K = 64, light_count, cells, lo[3], cell[3], inv_cell[3], band[3], margin[3]} (the last 15 are f32 bits), the
 * count of every cell then of the outside list (0xffffffff = overflow: every slot), then K slots per cell and K for the outside list
 * (0xffffffff past the count).  Cell (x, y, z) is index (z dims.y + y) dims.x + x.  While ST_OPT_TEXTURE_FILTER is on and a tick has
 * built them, "texture_mips" as 32-bit words: {T = pool texels, M = materials}, then per material 3 pairs {pool texel offset of level
 * 1, level count} for its base colour, emissive and metallic-roughness textures ({0, 0}: none; a count of 1: a 1x1 image, level 0
 * only), then the T
 * RGBA8 texels of the pool (byte 0 = red).  The pool holds levels 1.. of every live image in insertion order, level after level,
 * each row-major; level k + 1 is max(1, w_k >> 1) x max(1, h_k >> 1).  While the frames render with an environment map (set, and
 * taken by a tick), "environment_map" as 32-bit words: {W, H, intensity bits, rotation bits (reduced)}, then the W x H x 4 floats of
 * the texels as uploaded.  While ST_OPT_ENVIRONMENT_MAP_SAMPLING is on, a map is set and a tick has built its distribution,
 * "environment_map_distribution" as 32-bit words: {W, H, total bits}, then the H floats of the marginal CDF, then the H x W floats of
 * the conditional CDFs, row by row (the total is the marginal's last value; 0 or not finite: the frames do not use it). */
int st_read_scene(st_engine* e, const char* name, float* dst, size_t cap_floats, size_t* count);
int st_bvh_depth(st_engine* e, int* depth);
uint32_t st_frame(st_engine* e);
/* Sets the id of the frame the next st_tick prepares (ids start at 1, strolle/src/lib.rs:152).  Used by the
 * sample-parallel reference mode: rank g renders accumulations g+1, g+1+N, ... (SURVEY §8e, config C5). */
int st_set_frame(st_engine* e, uint32_t frame);
/* Ray-stream entry points (the ref_tracing / *_spatial_resampling::trace shape): `rays` = n x 8
 * host floats (origin.xyz, len, dir.xyz, pad).  closest: out = n x 12 floats (packed hit d0, d1
 * as in strolle-gpu/src/hit.rs:112-120, then distance, triangle id bits, material id bits,
 * used_memory).  any: out = n u32 flags.  `device_ms` (optional) receives kernel time. */
int st_trace_closest(st_engine* e, const float* rays, size_t n, float* out, float* device_ms);
int st_trace_any(st_engine* e, const float* rays, size_t n, uint32_t* out, float* device_ms);
/* elementary functions as evaluated on the device (op: 0 sin, 1 cos, 2 acos, 3 atan2, 4 exp, 5 pow, 6 glam's acos_approx, 7 the
 * flag-independent log2 of ST_OPT_TEXTURE_FILTER's level of detail, for finite a > 0, 8 and 9 the flag-independent acos and
 * atan2(a, b) of the environment map's lookup) */
int st_device_math(st_engine* e, int op, const float* a, const float* b, float* out, size_t n);
/* Per-pass device time (ms, CUDA events) accumulated since the last reset; `ms`/`launches`
 * have ST_PASS_COUNT entries indexed by st_pass_name(). */
#define ST_PASS_COUNT 27
int st_enable_timing(st_engine* e, int enabled);
int st_pass_times(st_engine* e, float* ms, uint32_t* launches, int reset);
const char* st_pass_name(int pass);
/* K22 frame_denoising::wavelet per à-trous iteration i (stride 2^i, strolle/src/camera_controller/passes/frame_denoising.rs:161-189):
 * device time (ms) and launches accumulated while timing is enabled; 5 entries each. */
int st_wavelet_times(st_engine* e, float* ms5, uint32_t* launches5, int reset);
/* Engine options.  ST_OPT_SVGF_FAST_MATH (default 1): the SVGF edge-stopping weights (K21/K22) use the
 * GPU's SFU approximations (ex2/sqrt/rcp.approx, <= 2 ulp) and fused multiply-adds, like a GLSL compiler
 * does for the reference's shaders; 0 selects strict IEEE arithmetic with polynomial exp, which makes the
 * denoiser bit-identical to the CPU oracle (everything else is bit-identical in both modes). */
enum { ST_OPT_SVGF_FAST_MATH = 1, ST_OPT_ASYNC_OUTPUT = 2, ST_OPT_HALO_NCCL = 3, ST_OPT_WAVELET_TILED = 4, ST_OPT_WAVELET_TILE_CFG = 5, ST_OPT_FUSE_REPROJECT = 6, ST_OPT_BVH_REUSE = 7, ST_OPT_VARIANCE_TILED = 8, ST_OPT_SHADING_FAST_MATH = 9, ST_OPT_STRIP_FUSED = 10, ST_OPT_FUSED_PASSES = 11, ST_OPT_STRIP_DMA = 12, ST_OPT_WAVELET_PAIRED = 13, ST_OPT_NORMAL_MAPS = 14, ST_OPT_BVH_REFIT = 15, ST_OPT_LIGHT_GRID = 16, ST_OPT_TEXTURE_FILTER = 17, ST_OPT_TEMPORAL_AA = 18, ST_OPT_ENVIRONMENT_MAP_SAMPLING = 19, ST_OPT_TONEMAPPING = 20, ST_OPT_AUTO_EXPOSURE = 21, ST_OPT_BLOOM = 22, ST_OPT_DEPTH_OF_FIELD = 23 };
/* ST_OPT_DEPTH_OF_FIELD (default 0; 1 = on, anything else is ST_ERR_INVALID): frames are defocused through a thin lens
 * (st_set_depth_of_field).  Once per rendered frame, after the composition or the temporal resolve and before the metering and the
 * bloom pyramid (timed as P_COMPOSITION), each pixel's signed circle-of-confusion radius r = clamp(k (z - F) / z, -R, R) is formed from
 * its view depth z (the primary hit distance of `surface_nd` times the cosine of its ray to the view axis; the sky takes min(k, R)),
 * and `output` is gathered over a disc of taps in 16 x 16 pixel tiles into a per-camera frame; a tile whose neighbourhood holds no
 * circle of 1/2 pixel or more is copied bit for bit.  That frame replaces `output` as the source of the Rgba32F copy, the metering
 * of ST_OPT_AUTO_EXPOSURE, the bloom pyramid and every Rgba8 store; `output` itself stays the sharp frame (temporal AA's history and
 * st_read_buffer("output") are unchanged), and st_copy_output never gathers again.  With F <= f the frame is not defocused (k = 0,
 * the frame is copied).  CameraMode::BvhHeatmap is not defocused.  Reference mode is not gathered: its depth-0 rays (K1, K2) leave a
 * thin lens instead, from a uniform point of the aperture disc of radius A / 2 on the camera's right and up axes towards the pinhole
 * ray's point at view depth F, drawn from a dispatch stream of its own, so that the accumulation converges to the thin-lens image; it
 * allocates no frame.  The frame is allocated zero-filled while the camera is defocused, freed when the option turns off, and reallocated when the camera is reallocated.
 * st_read_buffer("depth_of_field") returns, as 32-bit words: {W, H, TX, TY, defocused, f, A, k, F, R, forward.xyz, 0, 0, 0} (TX x TY
 * tiles; f .. forward as f32 bits), then r of every pixel (f32, row-major), then every tile's gather radius (u32, 0..32); it is
 * ST_ERR_NOT_FOUND while the camera is not defocused.  While the option is on, as set or as taken by the last st_tick,
 * st_render_strips and st_multi_render_camera over more than one member return ST_ERR_INVALID.  ST_STAT_DEPTH_OF_FIELD_GATHERS counts
 * the gathers.  Takes effect at the next st_tick. */
/* ST_OPT_BLOOM (default 0; 1 = on, anything else is ST_ERR_INVALID): the Rgba8UnormSrgb store gains a glow around bright light
 * (st_set_bloom).  After the frame is composed and metered (timed as P_COMPOSITION), once per rendered frame, a pyramid of `output` is
 * built: each channel cleared to 0 where it is not finite and > 0, times the exposure 2^(compensation - ev) while ST_OPT_TONEMAPPING is
 * not 0 (1 otherwise), through the soft-knee threshold, then L levels down (Jimenez's 13-tap filter, Karis-weighted on the first) and
 * back up (3 x 3 tent).  The store composites the glow B of level 0, brought to full resolution by the same tent, into the value it
 * would store (mode 0: (1 - intensity) x + intensity B, mode 1: x + intensity B), before T and today's store; st_copy_output
 * composites from the stored pyramid and never rebuilds it.  It applies to st_render_camera / st_copy_output with
 * ST_FORMAT_RGBA8_SRGB and the one-member st_multi_render_camera, with every ST_OPT_TONEMAPPING value; the Rgba32F frame and `output`
 * stay the linear, scene-referred frame, and CameraMode::BvhHeatmap is not bloomed.  The pyramid is allocated (zero-filled: a copy
 * before the first pyramid composites no glow) while the camera blooms, freed when the option turns off, and reallocated when the
 * camera is reallocated or `levels` changes.  st_read_buffer("bloom") returns it as the last rendered frame left it, as 32-bit words:
 * {L, w_0, h_0, .., w_7, h_7, 0, 0, 0} (level k is max(1, W >> (k + 1)) x max(1, H >> (k + 1)); zero past level L - 1), then
 * {r, g, b, 0} float texels, row-major: the down levels 0 .. L - 1, then the up levels 0 .. L - 2 (up_{L-1} is down_{L-1}).
 * While it is on, as set or as taken by the last st_tick, st_render_strips and st_multi_render_camera over more than one member return
 * ST_ERR_INVALID.  ST_STAT_BLOOM_PYRAMIDS counts the pyramid builds.  Takes effect at the next st_tick. */
/* ST_OPT_TONEMAPPING (default 0; 0..4, anything else is ST_ERR_INVALID): the display transform of the Rgba8UnormSrgb store.  0 keeps
 * today's store (clamp to [0, 1], sRGB OETF, round).  Otherwise each channel c of `output` becomes max(c, 0) (NaN -> 0) times
 * 2^(compensation - ev), goes through T, and is then stored as at 0.  T is 1: the identity (exposure only), 2: Reinhard on luminance,
 * x / (1 + L(x)), L = 0.2126 r + 0.7152 g + 0.0722 b, 3: ACES fitted (Hill's fit, as Bevy's AcesFitted), 4: AgX (the minimal AgX with
 * its 6th-order contrast polynomial, output as linear light).  It applies to st_render_camera / st_copy_output with
 * ST_FORMAT_RGBA8_SRGB and to the strip gathers; the Rgba32F frame and `output` stay the linear, scene-referred frame.
 * CameraMode::BvhHeatmap keeps today's store.  Takes effect at the next st_tick (DESIGN.md §2 "Exposure and tonemapping"). */
/* ST_OPT_AUTO_EXPOSURE (default 0; 1 = on, anything else is ST_ERR_INVALID; it has an effect only while ST_OPT_TONEMAPPING is not 0):
 * each camera meters its frame and adapts its own EV instead of taking st_exposure.ev.  After the frame is composed (timed as
 * P_COMPOSITION) a histogram of log2 L of `output` (256 bins of 1/8 stop over [-16, 16), pixels with a finite L > 0) is metered: the
 * pixels sorted by bin, the window [floor(low N), ceil(high N)) of the N counted is kept, its mean bin centre l gives the target
 * clamp(l - log2 0.18, ev_min, ev_max), and the EV moves toward it by at most speed_up per frame up and speed_down down (a first frame
 * jumps to it).  The metering runs once per rendered frame: st_copy_output does not meter.  The state is allocated while the camera
 * meters and restarts (a first frame) when metering turns on and when the camera is reallocated; st_read_buffer("exposure") returns it
 * as 32-bit words {ev, target (f32 bits), counted, kept, frames} then the 256 bin counts of the last frame.  The heat map is not
 * metered.  While it is on, st_render_strips and st_multi_render_camera over more than one member return ST_ERR_INVALID.
 * ST_STAT_EXPOSURE_METERINGS counts the metering launches.  Takes effect at the next st_tick. */
/* ST_OPT_ENVIRONMENT_MAP_SAMPLING (default 0; 1 = on, anything else is ST_ERR_INVALID): while an environment map is set
 * (st_set_environment_map), the GI bounce and the GI sky draw aim at the map's bright texels.  A tick that uploads a map with other
 * texels, or that finds the option turned on, builds on the device a distribution over the texels (weight: the largest RGB channel of
 * the texel's 3x3 neighbourhood times sin theta; f32 running sums, row by row, then over the rows); the distribution is freed when
 * the map is cleared or the option turns off.  With it, K12's bounce direction comes with probability 1/2 from the map and otherwise
 * from the BRDF, weighted by the mixture's density; K13's sky draw at a bounce hit comes from the map, weighted by its density.  Only
 * how directions are drawn changes, not what is estimated: the frame's expectation is the option-off one, with less variance where
 * the map's light is concentrated.  With no map, or a map whose total weight is 0 or not finite, every buffer is the option-off one.
 * Takes effect at the next st_tick; ST_STAT_ENVIRONMENT_MAP_DISTRIBUTION_BUILDS counts the builds; st_read_scene
 * ("environment_map_distribution") returns the distribution (DESIGN.md §2 "Environment map sampling"). */
/* ST_OPT_TEXTURE_FILTER (default 0; 1 = on, anything else is ST_ERR_INVALID): material textures are filtered through per-image mip
 * chains with a ray-cone level of detail, instead of the nearest texel of level 0 (the reference's sampler, so 0 keeps parity).
 * Level 0 is the image's atlas rect; levels 1.. (each texel the 2x2 box of the level above, averaged in linear light through the
 * sRGB table and re-encoded to the nearest byte; alpha averaged on the bytes) live in a device pool allocated only while the option
 * is on, rebuilt at st_tick when images or materials changed or the option turned on (ST_STAT_TEXTURE_MIP_BUILDS).  The level of
 * detail is lambda = 0.5 log2(A_uv W H w^2 |c| / (c.d)^2) for a hit on a triangle with edge cross product c and uv area A_uv, of
 * a W x H image, seen along d with cone width w: the spread of the pixel's camera ray to its right and lower neighbours at the
 * hit (primary hits), or a fresh cone from the segment's origin (the GI bounce, Reference mode at depth >= 1).  The sample is
 * trilinear: bilinear on levels floor(lambda) and floor(lambda) + 1 with repeat-wrapped taps inside the image.  It applies to base
 * colour, emissive and metallic-roughness at the G-buffer, to base colour and emissive at the GI bounce and in Reference mode; the
 * alpha test and normal maps keep the nearest level-0 texel.  Takes effect at the next st_tick (DESIGN.md §2). */
/* ST_OPT_TEMPORAL_AA (default 0; 1 = on, anything else is ST_ERR_INVALID): sub-pixel camera jitter and a temporal resolve.  Frame f
 * renders through J(f) = (h2(k) - 0.5, h3(k) - 0.5) pixels, k = ((f - 1) mod 16) + 1, h2 / h3 the base-2 / base-3 radical inverses
 * (in double, rounded to f32; screen y points down): pixel p's ray passes through the unjittered screen point p + 0.5 + J(f).  The
 * jitter is applied to the projection on the host (dx = -2 Jx / W, dy = 2 Jy / H; m[4c] += dx m[4c + 3], m[4c + 1] += dy m[4c + 3]
 * for every column c) before projection_view and ndc_to_world are derived, so every pass sees one consistent jittered camera; last
 * frame's camera is jittered with J(f - 1), J(0) = J(16).  Consequences: on a still camera the velocity map holds
 * -(J(f) - J(f - 1)), and st_read_buffer("curr_camera" / "prev_camera") returns the jittered cameras.  The composition step
 * (timed as P_COMPOSITION) then resolves instead of composing: per pixel the composed colour is tonemapped (c / (1 + max c)), the
 * history (Catmull-Rom at the surface's unjittered position last frame) is clipped into the 3x3 neighbourhood's YCoCg box and blended
 * with alpha = max(1 / (n + 1), 0.1), n the history's frame count (<= 16); `output` holds the resolved colour.  History lives in
 * "taa_history_a" / "taa_history_b" (st_read_buffer: tonemapped rgb, count), allocated while the option is on and reset by turning it
 * on and by camera reallocation.  Reference mode and CameraMode::BvhHeatmap are neither jittered nor resolved.  With the option on,
 * st_render_strips and st_multi_render_camera over more than one member return ST_ERR_INVALID.  ST_STAT_TAA_RESOLVES counts the
 * resolve launches.  Takes effect at the next st_tick (DESIGN.md §2). */
/* ST_OPT_LIGHT_GRID (default 0 = off; 1..64, anything else is ST_ERR_INVALID): the light candidates of ReSTIR DI sampling, of the GI
 * bounce's next-event estimate and of Reference mode are drawn uniformly from a per-cell list of the light slots that can reach the
 * point's cell, instead of from every slot.  N is the cell count along the longest axis of the grid box, the AABB of the range spheres of
 * the cullable lights (point lights with a finite position and colour and a range in [2^-60, 2^60]); the other axes get
 * max(1, ceil(N extent / longest)) cells.  A list holds, in ascending slot order, every non-cullable slot (the sun, spot lights, empty
 * slots) and every cullable light within range of the cell box grown by cell/64 + 8 ulp; outside the box a point samples the
 * non-cullable slots, and a non-finite point or a cell with more than 64 entries samples every slot, as with 0.  A dropped light's
 * radiance at any point of the cell is exactly zero, so the estimates stay unbiased: only the candidate count M and the noise change.
 * The lists are rebuilt on the device at st_tick whenever the lights were uploaded or the option changed (ST_STAT_LIGHT_GRID_BUILDS);
 * st_read_scene("light_grid") returns them.  The reference samples every slot, so the default keeps parity with it.  Takes effect at
 * the next st_tick (DESIGN.md §2). */
/* ST_OPT_BVH_REFIT (default 0): N > 0 allows up to N refit ticks in a row.  A refit tick is an st_tick whose only scene change is new
 * transforms of existing instances (same mesh, same material, nothing inserted or removed, no material's alpha mode changed): the moved
 * instances' triangles are baked on the device (bit-identical to the host bake) and the BVH boxes are recomputed bottom-up on the device
 * over the kept topology, with no host BVH build, no full upload and no stream synchronisation.  The next qualifying tick after N of
 * them, and every other instance change, rebuilds on the host as with 0.  After a refit the tree is no longer the one the reference
 * would build: closest hits stay the true closest hits (only equal-distance ties may resolve differently), any-hit answers are
 * unchanged, and CameraMode::BvhHeatmap / used_memory show the refit tree.  0 = every tick that changed an instance rebuilds, as the
 * reference does.  Takes effect at the next st_tick (DESIGN.md §2). */
/* ST_OPT_NORMAL_MAPS (default 0): materials with a normal map shade with the mapped normal, n' = normalize((t.x T + t.y B) + t.z N) with
 * t = 2 texel / 255 - 1, T the interpolated mesh tangent (not renormalised), B = w (N x T), w its handedness (mirrored instances flip
 * it); where n' is not finite (meshes without tangents) or n'.N <= 0 the interpolated normal N stays.  Back faces flip the result as
 * they flip N.  It reaches the G-buffer, the surface maps, the GI bounce hits and Reference mode's hits - everything shaded - but not
 * traversal, depth, velocity, triangle ids or the ray-stream entry points.  The reference ignores normal maps, so the default keeps
 * parity with it; while no material has a normal map the option changes nothing.  Takes effect at the next st_tick (DESIGN.md §2). */
/* ST_OPT_WAVELET_PAIRED (default 1; only with ST_OPT_SVGF_FAST_MATH, and never under the exchange-point strip transports, which ship the
 * named buffers between iterations): the wide-stride à-trous iterations, whose taps are scattered by the per-pixel jitter, read the DI and
 * GI signal as one interleaved 32-byte record per pixel (private scratch; one full sector per tap, loaded as two 128-bit loads on sm_90a,
 * instead of two half-used sectors).  1 = the stride-16 iteration reads records written by the stride-8 iteration; 2 = strides 8 and 16 both do (the
 * stride-4 iteration writes the records, the stride-8 iteration runs the gather kernel); 0 = planar buffers throughout.  On an H100 at
 * 1080p, 1 gives the fastest frame on Cornell and on the dungeon (DESIGN.md §4).  Same values in every layout; `*_diff_stash` then keeps
 * the output of the last planar iteration. */
#define ST_WAVELET_PAIRED_DEFAULT 1
/* ST_OPT_STRIP_DMA (fused strip transport only): which halos travel by copy engine (one side stream per neighbour, flag raised behind the
 * copy) instead of the producing kernel's own mirror stores.  1 = the 128-row halos of gi_reservoirs[1] / [2] (64 B per pixel, the bulk of
 * what travels), pushed right after the kernel that produced them and overlapping the DI passes that follow; 2 = also the 128 G-buffer rows
 * (prim_gbuffer_d0 / d1, surface map, surface_nd: 64 B per pixel) next to each strip edge right after the primary pass, instead of every
 * strip recomputing its neighbours' rows (which costs an inner strip of an 8-GPU frame two thirds of a G-buffer pass); 3 = also
 * di_reservoirs[1] and the preview pass's gi_reservoirs[3] (opt-in: the flags behind the copies arrive later than the in-kernel stores
 * do); 0 = every halo is mirrored in-kernel and the G-buffer rows are recomputed.
 * Default -1: level 1 for two strips (one neighbour: recomputing its rows is cheap), level 2 from three strips on. */
#define ST_STRIP_DMA_DEFAULT (-1)
/* ST_OPT_FUSED_PASSES (default 1): reference passes whose hand-over is private to a pixel or to a checkerboard pair run as ONE launch:
 * K5+K6 (di_sampling + di_temporal_resampling), K7+K8+K9 (di_spatial_resampling pick / trace / sample), K12+K13 (gi_sampling a + b),
 * K11 inside K14 on tracing frames (gi_reprojection + gi_temporal_resampling), K15+K16+K17 (gi_spatial_resampling) and the second
 * gi_preview_resampling pass + K19 gi_resolving.  Reservoirs, samples and every later buffer are bit-identical to the one-launch-per-
 * pass schedule; only the scratch textures between the fused members (and the intermediate gi_reservoirs entries they replaced) are no
 * longer written.  0 = one launch per reference dispatch (every buffer comparable with the oracle). */
#define ST_FUSED_PASSES_DEFAULT 1
/* ST_OPT_STRIP_FUSED (default 1): strip-partitioned frames use the fused transport (producer kernels store boundary rows straight
 * into the neighbours' buffers, neighbour-only sequence flags, halo rows of the G-buffer and of the SVGF chain recomputed instead of
 * shipped, DI / GI chains interleaved so that rows in flight overlap compute, temporal rows pulled on demand); 0 = one push +
 * all-rank barrier kernel per exchange point.  Needs strips of >= 128 rows. */
/* ST_OPT_SHADING_FAST_MATH (default 1): the ReSTIR DI/GI kernels K5-K19 (strolle-shaders/src/di_*.rs, gi_*.rs) run in their
 * fast-shading build: FMA contraction, approximate division / square root and SFU sin/cos/ex2/lg2 for radiance, BRDF, pdf
 * and MIS evaluation - the arithmetic a GPU shader compiler emits for the reference's SPIR-V.  BVH traversal, the ray/box and
 * ray/triangle tests, the alpha test and the RNG are identical in both builds (same hit for the same ray, bit for bit); the
 * frame stays inside the 1e-3 relative per-channel L2 tolerance.  0 = strict IEEE everywhere (bit-identical to the oracle). */
#define ST_SHADING_FAST_DEFAULT 1
/* ST_OPT_VARIANCE_TILED: 1 = K21 frame_denoising::estimate_variance (frame_denoising.rs:81-217) reads its 6x5 window from a
 * shared-memory tile filled by TMA tensor copies (identical results). */
#define ST_VARIANCE_TILED_DEFAULT 1
/* ST_OPT_BVH_REUSE (default 1): a BVH refresh takes over the subtrees of the previous tree whose primitive-centre
 * sequence is unchanged, as the reference does (strolle/src/bvh/builder.rs:245-275, hash = primitive.rs:27-37);
 * 0 = every refresh builds from scratch.  Both give the same tree unless a primitive changed while its centre did
 * not (e.g. only the instance's material): the reference keeps the old primitive in the reused leaf then (quirk C-20). */
/* ST_OPT_WAVELET_TILED: bit i set = à-trous iteration i (stride 2^i, K22 frame_denoising::wavelet,
 * strolle-shaders/src/frame_denoising.rs:220-361) runs the tile-staged kernel (pixel neighbourhood brought into
 * shared memory by TMA tensor copies) instead of the per-tap gather kernel; both produce identical bits.
 * ST_OPT_WAVELET_TILE_CFG: 4 bits per iteration, output-tile shape (0: 32x8, 1: 32x16, 2: 64x4, 3: 64x8 pixels). */
/* Defaults measured on an H100 at 1920x1080, Cornell and dungeon (DESIGN.md §4): strides 1, 2, 4, 8 tile-staged (32x8, 32x8, 32x8,
 * 32x16 output tiles), stride 16 gathers (its jittered 3x3 footprint does not fit a tile). */
#define ST_WAVELET_TILED_DEFAULT 15
#define ST_WAVELET_CFG_DEFAULT 0x01000
/* ST_OPT_FUSE_REPROJECT: 1 = K20 frame_denoising::reproject (frame_denoising.rs:4-78) handles the DI and the GI
 * signal in one launch (the reference dispatches it twice, passes/frame_denoising.rs:143-160); identical results. */
#define ST_FUSE_REPROJECT_DEFAULT 1
/* ST_OPT_HALO_NCCL (default 0): 1 keeps NCCL send/recv for the halo rows even when peer memory is linked. */
/* ST_OPT_ASYNC_OUTPUT (default 0): st_render_camera / st_copy_output only enqueue the device->host copy of
 * the composed frame and return; the caller keeps `host_out` (pinned) untouched until st_synchronize, and
 * alternates between two host buffers to pipeline frame N's copy with frame N+1's passes. */
int st_set_option(st_engine* e, int option, int value);
/* Engine statistics (development / test aid): tile-staged wavelet launches since creation, and how many of its
 * CTAs gave up waiting for their tensor copies (must stay 0). */
enum { ST_STAT_WAVELET_TILED_LAUNCHES = 1, ST_STAT_WAVELET_TILED_ERRORS = 2, ST_STAT_BVH_GRAFTED_SUBTREES = 3, ST_STAT_VARIANCE_TILED_LAUNCHES = 4,
       ST_STAT_STRIP_PULLED_ROWS = 5 /* rows x buffers fetched from other ranks by the temporal pull since linking */, ST_STAT_LAST_FRAME_FUSED_STRIPS = 6 /* 1 = the last strip frame used the fused transport */,
       ST_STAT_STRIP_FIRST_TIMEOUT = 7 /* 0, or 0x80000000 | slot << 16 | awaited rank << 8 | sequence & 0xff of the first strip flag wait that gave up */,
       ST_STAT_NORMAL_MAP_LAUNCHES = 8 /* launches of the normal-mapped kernel variants (ST_OPT_NORMAL_MAPS) since creation */,
       ST_STAT_BVH_REFITS = 9 /* refit ticks (ST_OPT_BVH_REFIT) since creation */,
       ST_STAT_LIGHT_GRID_BUILDS = 10 /* light grid builds (ST_OPT_LIGHT_GRID) since creation */,
       ST_STAT_TEXTURE_MIP_BUILDS = 11 /* mip-chain builds (ST_OPT_TEXTURE_FILTER) since creation */,
       ST_STAT_TAA_RESOLVES = 12 /* temporal resolve launches (ST_OPT_TEMPORAL_AA) since creation */,
       ST_STAT_ENVIRONMENT_MAP_LAUNCHES = 13 /* launches of the environment-mapped kernel variants (st_set_environment_map) since creation */,
       ST_STAT_ENVIRONMENT_MAP_DISTRIBUTION_BUILDS = 14 /* environment-map distribution builds (ST_OPT_ENVIRONMENT_MAP_SAMPLING) since creation */,
       ST_STAT_EXPOSURE_METERINGS = 15 /* metering launches (ST_OPT_AUTO_EXPOSURE) since creation */,
       ST_STAT_BLOOM_PYRAMIDS = 16 /* pyramid builds (ST_OPT_BLOOM) since creation */,
       ST_STAT_DEPTH_OF_FIELD_GATHERS = 17 /* depth-of-field gathers (ST_OPT_DEPTH_OF_FIELD) since creation */ };
int st_get_stat(st_engine* e, int stat, uint64_t* value);
/* The host-side BVH builder on its own (no device needed): binned-SAH build (strolle/src/bvh/builder.rs:17-319) + DFS
 * serialisation (serializer.rs:20-110) over `n` primitives of 11 floats each (triangle id bits, material id bits,
 * centre xyz, bounds min xyz, bounds max xyz; centre.x == FLT_MAX marks a dead primitive, primitive.rs:18-24).  The
 * builder object keeps the previous tree; `reuse` != 0 grafts its unchanged subtrees (builder.rs:245-359).  `out`
 * receives the float4 stream the GPU traverses (`*n_floats` floats); with out == NULL only the size is returned and
 * st_bvh_builder_read copies the stream of that build afterwards. */
typedef struct st_bvh_builder st_bvh_builder;
int st_bvh_builder_create(st_bvh_builder** out);
void st_bvh_builder_destroy(st_bvh_builder* b);
int st_bvh_builder_build(st_bvh_builder* b, const float* prims11, size_t n, int reuse, float* out, size_t cap_floats, size_t* n_floats,
                         uint32_t* grafted_subtrees, int* depth);
int st_bvh_builder_read(st_bvh_builder* b, float* out, size_t cap_floats);
/* external != 0: run the engine on the caller-owned CUDA stream `cuda_stream` (NULL = the legacy default
 * stream), e.g. the host runtime's stream that NCCL halo exchanges are ordered against; external == 0:
 * back to a private non-blocking stream. */
int st_set_stream(st_engine* e, void* cuda_stream, int external);
/* Ray statistics: counts executed Ray::trace / Ray::intersect calls (the Mrays/s numerator, SURVEY §8d). */
int st_count_rays(st_engine* e, int enabled);
int st_ray_count(st_engine* e, uint64_t* rays, int reset);
/* Native strip-parallel frame (SURVEY §8e): one engine per GPU/process, NCCL communicator owned by the engine.
 * rank 0 obtains an id (st_nccl_unique_id), the host runtime broadcasts the 128 bytes, every rank calls
 * st_nccl_init; st_render_strips then runs the frame's passes on this rank's row strip with an NCCL halo
 * exchange (grouped ncclSend/ncclRecv on the engine's stream) before each gathering pass, and, when `gather`
 * is non-zero (same value on every rank), assembles the composed frame on rank 0 in `format` (copied to `host_out`
 * there if non-NULL).  st_plan_frame exposes the exchange plan
 * ("step:buffer:reach;..." text) for tests. */
int st_nccl_unique_id(uint8_t* out128);
int st_nccl_init(st_engine* e, const uint8_t* id128, int rank, int world);
int st_plan_frame(const int* schedule, int n, uint32_t frame, int temporal_reach, char* out, size_t cap);
int st_render_strips(st_engine* e, st_camera_handle camera, void* host_out, int format, int temporal_reach, int gather);
/* The fused strip transport's order of one frame for a given pass schedule (st_frame_schedule), as text for tests:
 * "step:i;signal:SLOT:nb|all;wait:SLOT:nb|all[:prev];pull;push:buffer:SLOT;..." (no device needed).  `dma`: bits 0-1 = ST_OPT_STRIP_DMA (0, 1, 2),
 * bit 2 = a frame on which nothing moved (no temporal pull, no wait for PULL_DONE). */
int st_plan_strip_order(const int* schedule, int n, int dma, char* out, size_t cap);
/* The row partition st_render_strips / st_multi_* use for a frame of `height` rows over `world` ranks: rows_out[2r], rows_out[2r+1] = rank r's
 * [y0, y1).  Equal strips for one or two ranks; from three on the outer strips (one neighbour) get a few rows more than the inner ones
 * (two neighbours' worth of recomputed and mirrored halo rows).  No device needed. */
int st_strip_bounds(int height, int world, int* rows_out);
int st_halo_bytes(st_engine* e, uint64_t* bytes);
/* Peer-memory halo transport (default once linked): every rank exports CUDA IPC handles of the camera's buffers
 * (st_peer_export, ST_PEER_HANDLE_BYTES bytes), the host runtime all-gathers them, st_peer_import maps the other
 * ranks' buffers.  From then on st_render_strips replaces each NCCL exchange with ONE kernel that stores this
 * rank's boundary rows straight into the neighbours' buffers over NVLink, raises a sequence flag in every peer and
 * waits for theirs (a device-side barrier; no host involvement).  st_peer_errors counts barrier time-outs. */
#define ST_PEER_HANDLE_BYTES 192
int st_peer_export(st_engine* e, st_camera_handle camera, uint8_t* out192);
int st_peer_import(st_engine* e, st_camera_handle camera, const uint8_t* all_handles, int rank, int world);
int st_peer_errors(st_engine* e, st_camera_handle camera, uint32_t* count);
/* Device-side stopwatch on the engine's stream (CUDA events): st_mark_begin records, st_mark_end
 * records + waits and returns the elapsed milliseconds between the two. */
int st_mark_begin(st_engine* e);
int st_mark_end(st_engine* e, float* ms);
/* Row-strip partition for multi-GPU runs (SURVEY §8e): this engine computes rows [y0, y1) of the
 * camera's frame; full-frame buffers stay addressable for halo rows. */
int st_camera_set_strip(st_engine* e, st_camera_handle camera, int y0, int y1);
/* Device pointer + byte size of a per-camera buffer (for NCCL halo exchange by the host runtime). */
int st_buffer_device_ptr(st_engine* e, st_camera_handle camera, const char* name, void** ptr, size_t* bytes);
/* Stage-wise rendering for strip-parallel runs: executes passes [first, last] of the frame
 * schedule (indices into the schedule returned by st_frame_schedule). */
int st_frame_schedule(st_engine* e, st_camera_handle camera, int* pass_ids, int cap, int* count);
int st_render_range(st_engine* e, st_camera_handle camera, int first, int last);

/* Links engines of THIS process into one strip group (rank = index): enables peer access between their devices and maps every
 * member's per-camera buffers into the others (what st_peer_export / st_peer_import do between processes).  Members may share a
 * device (the whole protocol then runs on one GPU: how single-GPU boxes test it). */
int st_link_local(st_engine* const* engines, const st_camera_handle* cameras, int n);

/* ---- st_multi: one process, several devices (SURVEY 8b: `Engine::new` over a list of device ordinals) --------------------------
 * The strolle::Engine surface for a row-strip group: scene verbs are replayed on every member (the scene is replicated), a camera
 * exists on every member, st_multi_render_camera renders every member's strip of ONE frame with the fused transport and copies
 * each strip into the caller's frame.  Mirrors the st_* verbs one to one (lib.rs:132-301). */
typedef struct st_multi st_multi;
int st_multi_create(const int* device_ordinals, int n, st_multi** out);
void st_multi_destroy(st_multi* m);
int st_multi_size(st_multi* m);
st_engine* st_multi_engine(st_multi* m, int rank);   /* member access (statistics, options, st_read_buffer on one strip) */
st_camera_handle st_multi_member_camera(st_multi* m, st_camera_handle camera, int rank);
int st_multi_insert_mesh(st_multi* m, st_handle mesh, const st_mesh_triangle* triangles, size_t count);
int st_multi_remove_mesh(st_multi* m, st_handle mesh);
int st_multi_insert_material(st_multi* m, st_handle material, const st_material* mat);
int st_multi_has_material(st_multi* m, st_handle material);
int st_multi_remove_material(st_multi* m, st_handle material);
int st_multi_insert_image(st_multi* m, st_handle image, const uint8_t* rgba8, uint32_t width, uint32_t height);
int st_multi_remove_image(st_multi* m, st_handle image);
int st_multi_set_material_textures(st_multi* m, st_handle material, const st_material_textures* textures);
int st_multi_insert_instance(st_multi* m, st_handle instance, st_handle mesh, st_handle material, const float affine[12]);
int st_multi_remove_instance(st_multi* m, st_handle instance);
int st_multi_insert_light(st_multi* m, st_handle light, const st_light* l);
int st_multi_remove_light(st_multi* m, st_handle light);
int st_multi_update_sun(st_multi* m, float azimuth, float altitude);
int st_multi_set_environment_map(st_multi* m, const float* rgba32f, uint32_t width, uint32_t height, float intensity, float rotation);
int st_multi_create_camera(st_multi* m, const st_camera* camera, st_camera_handle* out);
int st_multi_update_camera(st_multi* m, st_camera_handle camera, const st_camera* desc);
int st_multi_delete_camera(st_multi* m, st_camera_handle camera);
int st_multi_tick(st_multi* m);
/* host_out: the full frame (width*height pixels of `format`); every member fills its own rows.  NULL = enqueue only. */
int st_multi_render_camera(st_multi* m, st_camera_handle camera, void* host_out, int format);
int st_multi_synchronize(st_multi* m);
int st_multi_set_option(st_multi* m, int option, int value);
int st_multi_set_exposure(st_multi* m, const st_exposure* exposure);
int st_multi_set_bloom(st_multi* m, const st_bloom* bloom);
int st_multi_set_depth_of_field(st_multi* m, const st_depth_of_field* dof);
int st_multi_set_seed_base(st_multi* m, uint32_t base);
int st_multi_set_blue_noise(st_multi* m, const uint8_t* rgba8_256x256);
int st_multi_read_buffer(st_multi* m, st_camera_handle camera, const char* name, float* dst, size_t cap_floats, size_t* count);
int st_multi_peer_errors(st_multi* m, st_camera_handle camera, uint32_t* count);

#ifdef __cplusplus
}
#endif
#endif /* STROLLE_B200_H */
