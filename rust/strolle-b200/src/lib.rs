//! `strolle::Engine<P>` on H100s.
//!
//! The public surface of the reference crate (`/strolle/src/lib.rs:104-409`: `Engine`, `Camera`, `CameraMode`, `CameraViewport`, `Mesh`,
//! `MeshTriangle`, `Material`, `AlphaMode`, `Light`, `Instance`, `Image`, `ImageData`, `Sun`, `Params`), with every method forwarding
//! to the C ABI of `libstrolle_b200.so` (`strolle-b200-sys`).  What differs, and why:
//!
//! * `Engine::new` takes CUDA device ordinals instead of a `&wgpu::Device`; one ordinal = one GPU, several = the frame is partitioned
//!   into row strips across them (`st_multi_*`).  `create_camera` / `update_camera` / `tick` lose their `device` / `queue` arguments.
//! * `render_camera` delivers the composed frame into a [`Frame`] (host pixels in the viewport's format) instead of recording into a
//!   wgpu command encoder — the CUDA kernels run on the engine's own stream.  A wgpu host uploads it with `Queue::write_texture`
//!   (what `bevy-strolle-b200` does), or reads the device pointer through `strolle_b200_sys::st_buffer_device_ptr` and interop.
//! * `ImageData::Texture` (a live wgpu texture) cannot be sampled from CUDA; dynamic images are passed as `ImageData::Raw` each time
//!   they change.
//! * Misuse returns `Err(Error)` where the reference panics (`triangles.rs:44-53`, `camera_controllers.rs:21-25`); the infallible
//!   scene verbs log the error and carry on like the reference's `warn!` paths (`images.rs:71-79`).
use std::collections::HashMap;
use std::ffi::CStr;
use std::fmt::{self, Debug};
use std::hash::Hash;
use std::marker::PhantomData;
use std::os::raw::c_int;

pub use glam;
use glam::{Affine3A, Mat4, UVec2, Vec2, Vec3, Vec4};
use strolle_b200_sys as sys;

/// Parameters used by Strolle to index textures, meshes etc. (`lib.rs:402-409`; `ImageTexture` has no CUDA meaning and is gone).
pub trait Params {
    type ImageHandle: Clone + Copy + Debug + Eq + Hash;
    type InstanceHandle: Clone + Copy + Debug + Eq + Hash;
    type LightHandle: Clone + Copy + Debug + Eq + Hash;
    type MaterialHandle: Clone + Copy + Debug + Eq + Hash;
    type MeshHandle: Clone + Copy + Debug + Eq + Hash;
}

#[derive(Clone, Debug)]
pub struct Error {
    pub code: i32,
    pub message: String,
}

impl fmt::Display for Error {
    fn fmt(&self, f: &mut fmt::Formatter<'_>) -> fmt::Result {
        write!(f, "strolle_b200 error {}: {}", self.code, self.message)
    }
}

impl std::error::Error for Error {}

fn check(code: c_int) -> Result<(), Error> {
    if code == sys::ST_OK {
        return Ok(());
    }
    let message = unsafe { CStr::from_ptr(sys::st_last_error()) }.to_string_lossy().into_owned();
    Err(Error { code, message })
}

fn soft(what: &str, code: c_int) {
    if let Err(err) = check(code) {
        log::warn!("{what}: {err}");
    }
}

// ---- scene types ------------------------------------------------------------------------------------------------------------------

/// `strolle::MeshTriangle` (`mesh_triangle.rs:7-45`)
#[derive(Clone, Debug, Default)]
pub struct MeshTriangle {
    positions: [Vec3; 3],
    normals: [Vec3; 3],
    uvs: [Vec2; 3],
    tangents: [Vec4; 3],
}

impl MeshTriangle {
    pub fn with_positions(mut self, positions: [impl Into<Vec3>; 3]) -> Self {
        self.positions = positions.map(Into::into);
        self
    }
    pub fn with_normals(mut self, normals: [impl Into<Vec3>; 3]) -> Self {
        self.normals = normals.map(Into::into);
        self
    }
    pub fn with_uvs(mut self, uvs: [impl Into<Vec2>; 3]) -> Self {
        self.uvs = uvs.map(Into::into);
        self
    }
    pub fn with_tangents(mut self, tangents: [impl Into<Vec4>; 3]) -> Self {
        self.tangents = tangents.map(Into::into);
        self
    }
    pub fn positions(&self) -> [Vec3; 3] {
        self.positions
    }
    pub fn normals(&self) -> [Vec3; 3] {
        self.normals
    }
    pub fn uvs(&self) -> [Vec2; 3] {
        self.uvs
    }
    fn to_ffi(&self) -> sys::st_mesh_triangle {
        sys::st_mesh_triangle {
            positions: self.positions.map(|v| v.to_array()),
            normals: self.normals.map(|v| v.to_array()),
            uvs: self.uvs.map(|v| v.to_array()),
            tangents: self.tangents.map(|v| v.to_array()),
        }
    }
}

/// `strolle::Mesh` (`mesh.rs:3-16`)
#[derive(Clone, Debug)]
pub struct Mesh {
    triangles: Vec<MeshTriangle>,
}

impl Mesh {
    pub fn new(triangles: Vec<MeshTriangle>) -> Self {
        Self { triangles }
    }
}

#[derive(Clone, Copy, Debug, Default, PartialEq, Eq)]
pub enum AlphaMode {
    #[default]
    Opaque,
    Blend,
}

/// `strolle::Material` (`material.rs:8-23`)
#[derive(Clone, Debug)]
pub struct Material<P: Params> {
    pub base_color: Vec4,
    pub base_color_texture: Option<P::ImageHandle>,
    pub emissive: Vec4,
    pub emissive_texture: Option<P::ImageHandle>,
    pub perceptual_roughness: f32,
    pub metallic: f32,
    pub metallic_roughness_texture: Option<P::ImageHandle>,
    pub reflectance: f32,
    pub ior: f32,
    pub normal_map_texture: Option<P::ImageHandle>,
    pub alpha_mode: AlphaMode,
}

impl<P: Params> Default for Material<P> {
    fn default() -> Self {
        Self {
            base_color: Vec4::ONE,
            base_color_texture: None,
            emissive: Vec4::ZERO,
            emissive_texture: None,
            perceptual_roughness: 0.5,
            metallic: 0.0,
            metallic_roughness_texture: None,
            reflectance: 0.5,
            ior: 1.0,
            normal_map_texture: None,
            alpha_mode: AlphaMode::Opaque,
        }
    }
}

/// `strolle::Light` (`light.rs:6-22`)
#[derive(Clone, Debug)]
pub enum Light {
    Point { position: Vec3, radius: f32, color: Vec3, range: f32 },
    Spot { position: Vec3, radius: f32, color: Vec3, range: f32, direction: Vec3, angle: f32 },
}

impl Light {
    fn to_ffi(&self) -> sys::st_light {
        match *self {
            Light::Point { position, radius, color, range } => sys::st_light {
                kind: sys::ST_LIGHT_POINT,
                position: position.to_array(),
                radius,
                color: color.to_array(),
                range,
                direction: [0.0; 3],
                angle: 0.0,
            },
            Light::Spot { position, radius, color, range, direction, angle } => sys::st_light {
                kind: sys::ST_LIGHT_SPOT,
                position: position.to_array(),
                radius,
                color: color.to_array(),
                range,
                direction: direction.to_array(),
                angle,
            },
        }
    }
}

/// `strolle::Instance` (`instance.rs:6-31`)
#[derive(Debug)]
pub struct Instance<P: Params> {
    mesh_handle: P::MeshHandle,
    material_handle: P::MaterialHandle,
    transform: Affine3A,
}

impl<P: Params> Instance<P> {
    pub fn new(mesh_handle: P::MeshHandle, material_handle: P::MaterialHandle, transform: Affine3A) -> Self {
        Self { mesh_handle, material_handle, transform }
    }
}

/// `strolle::ImageData::Raw` (`image.rs:36-47`): tightly packed RGBA8 texels of an `Rgba8UnormSrgb` image
#[derive(Debug)]
pub enum ImageData {
    Raw { data: Vec<u8> },
}

/// `strolle::Image` (`image.rs:3-34`)
#[derive(Debug)]
pub struct Image {
    data: ImageData,
    size: UVec2,
}

impl Image {
    pub fn new(data: ImageData, size: UVec2) -> Self {
        Self { data, size }
    }
}

/// An equirectangular environment map of linear RGB that lights the scene in place of the procedural sky: `width` x `height`
/// texels, row-major, row 0 the zenith (alpha ignored); with `rotation` 0 the centre column is seen looking down -Z.  The radiance is
/// the bilinear blend times `intensity`.  See `st_set_environment_map` in include/strolle_b200.h.
#[derive(Clone, Debug, PartialEq)]
pub struct EnvironmentMap {
    pub width: u32,
    pub height: u32,
    pub texels: Vec<[f32; 4]>,
    pub intensity: f32,
    pub rotation: f32,
}

/// `strolle::Sun` (`sun.rs:1-14`)
#[derive(Clone, Copy, Debug, PartialEq)]
pub struct Sun {
    pub azimuth: f32,
    pub altitude: f32,
}

impl Default for Sun {
    fn default() -> Self {
        Self { azimuth: 0.0, altitude: 0.35 }
    }
}

// ---- cameras ----------------------------------------------------------------------------------------------------------------------

/// `strolle::CameraMode` (`camera.rs:83-105`)
#[derive(Clone, Copy, Debug, PartialEq, Eq)]
pub enum CameraMode {
    Image { denoise: bool },
    DiDiffuse { denoise: bool },
    DiSpecular { denoise: bool },
    GiDiffuse { denoise: bool },
    GiSpecular { denoise: bool },
    BvhHeatmap,
    Reference { depth: u8 },
}

impl Default for CameraMode {
    fn default() -> Self {
        Self::Image { denoise: true }
    }
}

/// The display transform of `Rgba8UnormSrgb` frames (`ST_OPT_TONEMAPPING`), applied after the exposure.
#[derive(Clone, Copy, Debug, Default, PartialEq, Eq)]
pub enum Tonemapping {
    /// Linear light clamped to [0, 1] (the reference's store).
    #[default]
    None = 0,
    /// The exposure only.
    Exposure = 1,
    /// Reinhard on luminance, x / (1 + L(x)).
    Reinhard = 2,
    /// Hill's fit of ACES, as Bevy's `AcesFitted`.
    AcesFitted = 3,
    /// The minimal AgX with its 6th-order contrast polynomial.
    AgX = 4,
}

/// The exposure of tonemapped frames, in stops (`st_exposure`): the stored value is the scene value times 2^(compensation - ev).
#[derive(Clone, Copy, Debug, PartialEq)]
pub struct Exposure {
    /// Manual exposure (auto exposure off).
    pub ev: f32,
    /// Added in both modes.
    pub compensation: f32,
    /// Clamp on the metered EV.
    pub ev_min: f32,
    pub ev_max: f32,
    /// The metered fraction of the pixels: the darkest `low` and the brightest `1 - high` are dropped.
    pub low: f32,
    pub high: f32,
    /// Largest EV change per frame, up and down.
    pub speed_up: f32,
    pub speed_down: f32,
}

impl Default for Exposure {
    fn default() -> Self {
        Self { ev: 0.0, compensation: 0.0, ev_min: -8.0, ev_max: 8.0, low: 0.1, high: 0.9, speed_up: 0.05, speed_down: 1.0 / 60.0 }
    }
}

/// How the glow enters the stored value (`st_bloom::mode`).
#[derive(Clone, Copy, Debug, Default, PartialEq, Eq)]
pub enum BloomMode {
    /// (1 - intensity) x + intensity B: a constant frame stays constant; `intensity` in [0, 1].
    #[default]
    EnergyConserving = 0,
    /// x + intensity B; `intensity` >= 0.
    Additive = 1,
}

/// The glow around bright light in `Rgba8UnormSrgb` frames (`st_bloom`, `ST_OPT_BLOOM`): a downsample / upsample pyramid of the
/// exposed frame, composited before the display transform.
#[derive(Clone, Copy, Debug, PartialEq)]
pub struct Bloom {
    /// The glow's share of the stored value.
    pub intensity: f32,
    /// How far the glow spreads, in [0, 1]: level k of the pyramid weighs (1 - scatter) scatter^k.
    pub scatter: f32,
    /// The exposed brightness (largest channel) where the glow starts; 0 lets every pixel glow.
    pub threshold: f32,
    /// The soft knee's width as a fraction of the threshold, in [0, 1].
    pub softness: f32,
    /// The pyramid's depth, 1..=8; level 0 is half resolution.
    pub levels: i32,
    pub mode: BloomMode,
}

impl Default for Bloom {
    fn default() -> Self {
        Self { intensity: 0.15, scatter: 0.7, threshold: 0.0, softness: 0.0, levels: 7, mode: BloomMode::EnergyConserving }
    }
}

/// The thin lens of defocused frames (`st_depth_of_field`, `ST_OPT_DEPTH_OF_FIELD`): a circle-of-confusion gather of each frame.
#[derive(Clone, Copy, Debug, PartialEq)]
pub struct DepthOfField {
    /// The view depth in focus, in scene units (> 0).
    pub focal_distance: f32,
    /// The f-number (> 0): the aperture's diameter is the focal length over it.
    pub aperture_f_stops: f32,
    /// The sensor's height in scene units (> 0); with the projection's vertical field of view it gives the focal length.
    pub sensor_height: f32,
    /// The largest radius of the circle of confusion, in output pixels, in [1, 32].
    pub max_radius: f32,
}

impl Default for DepthOfField {
    fn default() -> Self {
        Self { focal_distance: 10.0, aperture_f_stops: 1.0, sensor_height: 0.01866, max_radius: 16.0 }
    }
}

/// The two formats the engine composes into (`CameraViewport::format`, `camera.rs:170-185`)
#[derive(Clone, Copy, Debug, PartialEq, Eq)]
pub enum ViewportFormat {
    Rgba8UnormSrgb,
    Rgba32Float,
}

impl ViewportFormat {
    pub fn bytes_per_pixel(self) -> usize {
        match self {
            Self::Rgba8UnormSrgb => 4,
            Self::Rgba32Float => 16,
        }
    }
    fn to_ffi(self) -> c_int {
        match self {
            Self::Rgba8UnormSrgb => sys::ST_FORMAT_RGBA8_SRGB,
            Self::Rgba32Float => sys::ST_FORMAT_RGBA32F,
        }
    }
}

#[derive(Clone, Debug)]
pub struct CameraViewport {
    pub format: ViewportFormat,
    pub size: UVec2,
    pub position: UVec2,
}

impl Default for CameraViewport {
    fn default() -> Self {
        Self { format: ViewportFormat::Rgba8UnormSrgb, size: UVec2::new(512, 512), position: UVec2::ZERO }
    }
}

/// `strolle::Camera` (`camera.rs:8-14`)
#[derive(Clone, Debug, Default)]
pub struct Camera {
    pub mode: CameraMode,
    pub viewport: CameraViewport,
    pub transform: Mat4,
    pub projection: Mat4,
}

impl Camera {
    fn to_ffi(&self) -> sys::st_camera {
        let (mode, denoise, ref_depth) = match self.mode {
            CameraMode::Image { denoise } => (sys::ST_MODE_IMAGE, denoise, 0),
            CameraMode::DiDiffuse { denoise } => (sys::ST_MODE_DI_DIFFUSE, denoise, 0),
            CameraMode::DiSpecular { denoise } => (sys::ST_MODE_DI_SPECULAR, denoise, 0),
            CameraMode::GiDiffuse { denoise } => (sys::ST_MODE_GI_DIFFUSE, denoise, 0),
            CameraMode::GiSpecular { denoise } => (sys::ST_MODE_GI_SPECULAR, denoise, 0),
            CameraMode::BvhHeatmap => (sys::ST_MODE_BVH_HEATMAP, false, 0),
            CameraMode::Reference { depth } => (sys::ST_MODE_REFERENCE, false, depth as i32),
        };
        sys::st_camera {
            mode,
            denoise: denoise as i32,
            ref_depth,
            width: self.viewport.size.x,
            height: self.viewport.size.y,
            transform: self.transform.to_cols_array(),
            projection: self.projection.to_cols_array(),
        }
    }
}

#[derive(Clone, Copy, Debug, PartialEq, Eq, Hash)]
pub struct CameraHandle(sys::st_camera_handle);

/// Host pixels of one composed frame, `viewport.size.x * viewport.size.y` texels of `format`, row-major.  Allocate once per camera
/// (page-locked memory makes the device-to-host copy asynchronous and full speed) and reuse.
#[derive(Debug)]
pub struct Frame {
    pub format: ViewportFormat,
    pub size: UVec2,
    pub pixels: Vec<u8>,
}

impl Frame {
    pub fn new(viewport: &CameraViewport) -> Self {
        let n = viewport.size.x as usize * viewport.size.y as usize * viewport.format.bytes_per_pixel();
        Self { format: viewport.format, size: viewport.size, pixels: vec![0; n] }
    }
}

// ---- engine -----------------------------------------------------------------------------------------------------------------------

/// Maps the host's own handle types (`P::*Handle`) to the opaque `u64` handles of the C ABI.
#[derive(Debug)]
struct Interner<H: Copy + Eq + Hash> {
    ids: HashMap<H, u64>,
    next: u64,
}

impl<H: Copy + Eq + Hash> Default for Interner<H> {
    fn default() -> Self {
        Self { ids: HashMap::new(), next: 1 }
    }
}

impl<H: Copy + Eq + Hash> Interner<H> {
    fn id(&mut self, handle: H) -> u64 {
        if let Some(id) = self.ids.get(&handle) {
            return *id;
        }
        let id = self.next;
        self.next += 1;
        self.ids.insert(handle, id);
        id
    }
    fn get(&self, handle: H) -> Option<u64> {
        self.ids.get(&handle).copied()
    }
    fn forget(&mut self, handle: H) -> Option<u64> {
        self.ids.remove(&handle)
    }
}

/// `strolle::Engine<P>` (`lib.rs:104-395`) over one or several GPUs.
pub struct Engine<P: Params> {
    raw: *mut sys::st_multi,
    meshes: Interner<P::MeshHandle>,
    materials: Interner<P::MaterialHandle>,
    images: Interner<P::ImageHandle>,
    instances: Interner<P::InstanceHandle>,
    lights: Interner<P::LightHandle>,
    viewports: HashMap<CameraHandle, CameraViewport>,
    _params: PhantomData<P>,
}

// The C ABI is externally synchronised (single writer) like `ResMut<Engine>` in the host; the raw pointer is not aliased.
unsafe impl<P: Params> Send for Engine<P> {}
unsafe impl<P: Params> Sync for Engine<P> {}

impl<P: Params> Debug for Engine<P> {
    fn fmt(&self, f: &mut fmt::Formatter<'_>) -> fmt::Result {
        write!(f, "Engine({} device(s))", unsafe { sys::st_multi_size(self.raw) })
    }
}

impl<P: Params> Engine<P> {
    /// `Engine::new` (`lib.rs:132-158`).  `devices` = CUDA ordinals; more than one partitions every camera's frame into row strips.
    pub fn new(devices: &[i32]) -> Result<Self, Error> {
        log::info!("Initializing on CUDA device(s) {devices:?}");
        let mut raw = std::ptr::null_mut();
        check(unsafe { sys::st_multi_create(devices.as_ptr(), devices.len() as c_int, &mut raw) })?;
        // the 256x256 RGBA8 blue-noise tile the reference embeds as a PNG (`noise.rs:30-66`, strolle/assets/blue-noise.png)
        static BLUE_NOISE: &[u8] = include_bytes!("../../../strolle_b200/assets/blue_noise_256_rgba8.bin");
        check(unsafe { sys::st_multi_set_blue_noise(raw, BLUE_NOISE.as_ptr()) })?;
        Ok(Self {
            raw,
            meshes: Default::default(),
            materials: Default::default(),
            images: Default::default(),
            instances: Default::default(),
            lights: Default::default(),
            viewports: HashMap::new(),
            _params: PhantomData,
        })
    }

    /// Shades with the materials' normal maps (`ST_OPT_NORMAL_MAPS`, off by default: the reference ignores them).  Takes effect
    /// with the next frame's scene update.
    pub fn set_normal_maps(&mut self, on: bool) -> Result<(), Error> {
        check(unsafe { sys::st_multi_set_option(self.raw, sys::ST_OPT_NORMAL_MAPS, on as c_int) })
    }

    /// Lets up to `ticks` frames in a row that only move instances refit the BVH on the GPU instead of rebuilding it on the host
    /// (`ST_OPT_BVH_REFIT`; 0, the default, rebuilds every time, as the reference does).  Takes effect with the next frame's scene update.
    pub fn set_bvh_refit(&mut self, ticks: u32) -> Result<(), Error> {
        check(unsafe { sys::st_multi_set_option(self.raw, sys::ST_OPT_BVH_REFIT, ticks.min(c_int::MAX as u32) as c_int) })
    }

    /// Draws the light candidates from a world-space grid of the lights that can reach each cell, `cells` cells along its longest
    /// axis (`ST_OPT_LIGHT_GRID`, 1..=64; 0, the default, draws from every light, as the reference does).  Takes effect with the next
    /// frame's scene update.
    pub fn set_light_grid(&mut self, cells: u32) -> Result<(), Error> {
        check(unsafe { sys::st_multi_set_option(self.raw, sys::ST_OPT_LIGHT_GRID, cells.min(c_int::MAX as u32) as c_int) })
    }

    /// Filters material textures through per-image mip chains with a ray-cone level of detail (`ST_OPT_TEXTURE_FILTER`; off, the
    /// default, takes the nearest texel, as the reference does).  Takes effect with the next frame's scene update.
    pub fn set_texture_filter(&mut self, on: bool) -> Result<(), Error> {
        check(unsafe { sys::st_multi_set_option(self.raw, sys::ST_OPT_TEXTURE_FILTER, on as c_int) })
    }

    /// Anti-aliases frames with sub-pixel camera jitter and a temporal resolve in place of the frame composition
    /// (`ST_OPT_TEMPORAL_AA`; off, the default, renders one ray through each pixel centre, as the reference does).  Needs an engine
    /// over one device: row strips over several refuse to render while it is on.  Takes effect with the next frame's scene update.
    pub fn set_temporal_aa(&mut self, on: bool) -> Result<(), Error> {
        check(unsafe { sys::st_multi_set_option(self.raw, sys::ST_OPT_TEMPORAL_AA, on as c_int) })
    }

    /// Draws the GI bounce and the GI sky draw from the environment map's distribution, where its light is
    /// (`ST_OPT_ENVIRONMENT_MAP_SAMPLING`; off, the default, draws from the BRDF and the uniform hemisphere, as the reference does).
    /// Changes only the noise, not the expected frame; has an effect only while a map is set.  Takes effect with the next frame's
    /// scene update.
    pub fn set_environment_map_sampling(&mut self, on: bool) -> Result<(), Error> {
        check(unsafe { sys::st_multi_set_option(self.raw, sys::ST_OPT_ENVIRONMENT_MAP_SAMPLING, on as c_int) })
    }

    /// The display transform of `Rgba8UnormSrgb` frames (`ST_OPT_TONEMAPPING`; `Tonemapping::None`, the default, clamps linear light
    /// to [0, 1], as the reference does).  `Rgba32Float` frames stay linear and scene-referred.  Takes effect with the next frame's
    /// scene update.
    pub fn set_tonemapping(&mut self, t: Tonemapping) -> Result<(), Error> {
        check(unsafe { sys::st_multi_set_option(self.raw, sys::ST_OPT_TONEMAPPING, t as c_int) })
    }

    /// Each camera meters its frame and adapts its own EV (`ST_OPT_AUTO_EXPOSURE`; off, the default, takes `Exposure::ev`).  Has an
    /// effect only while the tonemapping is not `Tonemapping::None`; needs an engine over one device: row strips over several refuse
    /// to render while it is on.  Takes effect with the next frame's scene update.
    pub fn set_auto_exposure(&mut self, on: bool) -> Result<(), Error> {
        check(unsafe { sys::st_multi_set_option(self.raw, sys::ST_OPT_AUTO_EXPOSURE, on as c_int) })
    }

    /// The exposure of tonemapped frames (`st_set_exposure`); refused as a whole when a field is out of range.  Takes effect with the
    /// next frame's scene update.
    pub fn set_exposure(&mut self, e: &Exposure) -> Result<(), Error> {
        let x = sys::st_exposure {
            ev: e.ev, compensation: e.compensation, ev_min: e.ev_min, ev_max: e.ev_max, low: e.low, high: e.high, speed_up: e.speed_up,
            speed_down: e.speed_down,
        };
        check(unsafe { sys::st_multi_set_exposure(self.raw, &x) })
    }

    /// A glow around bright light in `Rgba8UnormSrgb` frames (`ST_OPT_BLOOM` and `st_set_bloom`; `None`, the default, stores no glow).
    /// It works with every tonemapping, `Tonemapping::None` included; `Rgba32Float` frames stay linear and without glow.  Needs an
    /// engine over one device: row strips over several refuse to render while it is on.  Refused as a whole when a field is out of
    /// range.  Takes effect with the next frame's scene update.
    pub fn set_bloom(&mut self, bloom: Option<&Bloom>) -> Result<(), Error> {
        if let Some(b) = bloom {
            let x = sys::st_bloom {
                intensity: b.intensity, scatter: b.scatter, threshold: b.threshold, softness: b.softness, levels: b.levels, mode: b.mode as i32,
            };
            check(unsafe { sys::st_multi_set_bloom(self.raw, &x) })?;
        }
        check(unsafe { sys::st_multi_set_option(self.raw, sys::ST_OPT_BLOOM, bloom.is_some() as c_int) })
    }

    /// Defocuses frames through a thin lens (`ST_OPT_DEPTH_OF_FIELD` and `st_set_depth_of_field`; `None`, the default, keeps every
    /// frame sharp).  Both frame formats show the defocused frame; Reference mode samples the lens in its primary rays; the heat map stays sharp.  Needs an engine over one
    /// device: row strips over several refuse to render while it is on.  Refused as a whole when a field is out of range.  Takes effect
    /// with the next frame's scene update.
    pub fn set_depth_of_field(&mut self, dof: Option<&DepthOfField>) -> Result<(), Error> {
        if let Some(d) = dof {
            let x = sys::st_depth_of_field {
                focal_distance: d.focal_distance, aperture_f_stops: d.aperture_f_stops, sensor_height: d.sensor_height, max_radius: d.max_radius,
            };
            check(unsafe { sys::st_multi_set_depth_of_field(self.raw, &x) })?;
        }
        check(unsafe { sys::st_multi_set_option(self.raw, sys::ST_OPT_DEPTH_OF_FIELD, dof.is_some() as c_int) })
    }

    /// Lights the scene from an equirectangular environment map in place of the procedural sky (`st_set_environment_map`; `None`,
    /// the default, keeps the reference's procedural sky).  The sun light still follows `update_sun`: to light from the map alone,
    /// put the sun below the horizon.  Takes effect with the next frame's scene update.
    pub fn set_environment_map(&mut self, map: Option<&EnvironmentMap>) -> Result<(), Error> {
        match map {
            None => check(unsafe { sys::st_multi_set_environment_map(self.raw, std::ptr::null(), 0, 0, 0.0, 0.0) }),
            Some(m) => {
                if m.texels.len() as u64 != m.width as u64 * m.height as u64 {
                    return Err(Error { code: sys::ST_ERR_INVALID, message: "environment map: texels.len() != width * height".into() });
                }
                check(unsafe {
                    sys::st_multi_set_environment_map(self.raw, m.texels.as_ptr() as *const f32, m.width, m.height, m.intensity, m.rotation)
                })
            }
        }
    }

    /// Creates or updates a mesh (`lib.rs:161-164`).
    pub fn insert_mesh(&mut self, handle: P::MeshHandle, item: Mesh) {
        let id = self.meshes.id(handle);
        let tris: Vec<sys::st_mesh_triangle> = item.triangles.iter().map(MeshTriangle::to_ffi).collect();
        soft("insert_mesh", unsafe { sys::st_multi_insert_mesh(self.raw, id, tris.as_ptr(), tris.len()) });
    }

    /// Removes a mesh (`lib.rs:166-171`); instances that refer to it are not removed.
    pub fn remove_mesh(&mut self, handle: P::MeshHandle) {
        if let Some(id) = self.meshes.forget(handle) {
            soft("remove_mesh", unsafe { sys::st_multi_remove_mesh(self.raw, id) });
        }
    }

    /// Creates or updates a material (`lib.rs:174-181`).
    pub fn insert_material(&mut self, handle: P::MaterialHandle, item: Material<P>) {
        let id = self.materials.id(handle);
        let ffi = sys::st_material {
            base_color: item.base_color.to_array(),
            emissive: item.emissive.to_array(),
            perceptual_roughness: item.perceptual_roughness,
            metallic: item.metallic,
            reflectance: item.reflectance,
            ior: item.ior,
            alpha_blend: (item.alpha_mode == AlphaMode::Blend) as i32,
        };
        soft("insert_material", unsafe { sys::st_multi_insert_material(self.raw, id, &ffi) });
        let slots = [item.base_color_texture, item.emissive_texture, item.metallic_roughness_texture, item.normal_map_texture];
        let mut tex = sys::st_material_textures::default();
        let mut ids = [0u64; 4];
        for (k, slot) in slots.iter().enumerate() {
            if let Some(image) = slot {
                ids[k] = self.images.id(*image);
                tex.mask |= 1 << k;
            }
        }
        tex.base_color = ids[0];
        tex.emissive = ids[1];
        tex.metallic_roughness = ids[2];
        tex.normal_map = ids[3];
        soft("insert_material (textures)", unsafe { sys::st_multi_set_material_textures(self.raw, id, &tex) });
    }

    /// Returns whether given material exists (`lib.rs:184-186`).
    pub fn has_material(&self, handle: P::MaterialHandle) -> bool {
        match self.materials.get(handle) {
            Some(id) => unsafe { sys::st_multi_has_material(self.raw, id) != 0 },
            None => false,
        }
    }

    /// Removes a material (`lib.rs:192-195`).
    pub fn remove_material(&mut self, handle: P::MaterialHandle) {
        if let Some(id) = self.materials.forget(handle) {
            soft("remove_material", unsafe { sys::st_multi_remove_material(self.raw, id) });
        }
    }

    /// Creates or updates an image (`lib.rs:198-205`).
    pub fn insert_image(&mut self, handle: P::ImageHandle, image: Image) {
        let id = self.images.id(handle);
        let ImageData::Raw { data } = &image.data;
        let expected = image.size.x as usize * image.size.y as usize * 4;
        if data.len() != expected {
            log::warn!("insert_image: {} bytes given, {}x{} RGBA8 needs {expected}; image skipped", data.len(), image.size.x, image.size.y);
            return;
        }
        soft("insert_image", unsafe { sys::st_multi_insert_image(self.raw, id, data.as_ptr(), image.size.x, image.size.y) });
    }

    /// Removes an image (`lib.rs:211-214`).
    pub fn remove_image(&mut self, handle: P::ImageHandle) {
        if let Some(id) = self.images.forget(handle) {
            soft("remove_image", unsafe { sys::st_multi_remove_image(self.raw, id) });
        }
    }

    /// Creates or updates an instance (`lib.rs:217-223`).
    pub fn insert_instance(&mut self, handle: P::InstanceHandle, instance: Instance<P>) {
        let id = self.instances.id(handle);
        let mesh = self.meshes.id(instance.mesh_handle);
        let material = self.materials.id(instance.material_handle);
        let m = instance.transform.matrix3;
        let t = instance.transform.translation;
        let affine = [m.x_axis.x, m.x_axis.y, m.x_axis.z, m.y_axis.x, m.y_axis.y, m.y_axis.z, m.z_axis.x, m.z_axis.y, m.z_axis.z, t.x, t.y, t.z];
        soft("insert_instance", unsafe { sys::st_multi_insert_instance(self.raw, id, mesh, material, affine.as_ptr()) });
    }

    /// Removes an instance (`lib.rs:226-229`).
    pub fn remove_instance(&mut self, handle: P::InstanceHandle) {
        if let Some(id) = self.instances.forget(handle) {
            soft("remove_instance", unsafe { sys::st_multi_remove_instance(self.raw, id) });
        }
    }

    /// Creates or updates a light (`lib.rs:232-234`).
    pub fn insert_light(&mut self, handle: P::LightHandle, item: Light) {
        let id = self.lights.id(handle);
        soft("insert_light", unsafe { sys::st_multi_insert_light(self.raw, id, &item.to_ffi()) });
    }

    /// Removes a light (`lib.rs:237-239`).
    pub fn remove_light(&mut self, handle: P::LightHandle) {
        if let Some(id) = self.lights.forget(handle) {
            soft("remove_light", unsafe { sys::st_multi_remove_light(self.raw, id) });
        }
    }

    /// Updates sun's parameters (`lib.rs:242-245`).
    pub fn update_sun(&mut self, sun: Sun) {
        soft("update_sun", unsafe { sys::st_multi_update_sun(self.raw, sun.azimuth, sun.altitude) });
    }

    /// Creates a new camera (`lib.rs:252-259`): allocates its per-camera buffers on every device of the group.
    pub fn create_camera(&mut self, camera: Camera) -> Result<CameraHandle, Error> {
        let mut out = 0;
        check(unsafe { sys::st_multi_create_camera(self.raw, &camera.to_ffi(), &mut out) })?;
        let handle = CameraHandle(out);
        self.viewports.insert(handle, camera.viewport);
        Ok(handle)
    }

    /// Updates camera, changing its mode, position, size etc. (`lib.rs:262-273`).
    pub fn update_camera(&mut self, handle: CameraHandle, camera: Camera) -> Result<(), Error> {
        check(unsafe { sys::st_multi_update_camera(self.raw, handle.0, &camera.to_ffi()) })?;
        self.viewports.insert(handle, camera.viewport);
        Ok(())
    }

    /// Renders camera (`lib.rs:279-286`) and delivers the composed frame into `target`, whose format and size must be the
    /// viewport's.  Returns once the pixels are in `target`.
    pub fn render_camera(&self, handle: CameraHandle, target: &mut Frame) -> Result<(), Error> {
        let viewport = self.viewports.get(&handle).ok_or_else(|| Error { code: sys::ST_ERR_NOT_FOUND, message: "unknown camera".into() })?;
        if target.format != viewport.format || target.size != viewport.size {
            return Err(Error { code: sys::ST_ERR_INVALID, message: "target frame does not match the camera's viewport".into() });
        }
        check(unsafe { sys::st_multi_render_camera(self.raw, handle.0, target.pixels.as_mut_ptr().cast(), target.format.to_ffi()) })
    }

    /// Enqueues the camera's passes without reading the frame back (e.g. `CameraMode::Reference` accumulation frames).
    pub fn render_camera_offscreen(&self, handle: CameraHandle) -> Result<(), Error> {
        check(unsafe { sys::st_multi_render_camera(self.raw, handle.0, std::ptr::null_mut(), sys::ST_FORMAT_RGBA32F) })
    }

    /// Deletes a camera (`lib.rs:292-294`).
    pub fn delete_camera(&mut self, handle: CameraHandle) -> Result<(), Error> {
        self.viewports.remove(&handle);
        check(unsafe { sys::st_multi_delete_camera(self.raw, handle.0) })
    }

    /// Sends all changes to the GPUs and prepares them for the upcoming frame (`lib.rs:301-395`); call once per frame before
    /// [`Self::render_camera`].
    pub fn tick(&mut self) -> Result<(), Error> {
        check(unsafe { sys::st_multi_tick(self.raw) })
    }

    /// Engine options of the C ABI (`ST_OPT_*`), applied to every device.
    pub fn set_option(&mut self, option: i32, value: i32) -> Result<(), Error> {
        check(unsafe { sys::st_multi_set_option(self.raw, option, value) })
    }
}

impl<P: Params> Drop for Engine<P> {
    fn drop(&mut self) {
        unsafe { sys::st_multi_destroy(self.raw) };
    }
}
