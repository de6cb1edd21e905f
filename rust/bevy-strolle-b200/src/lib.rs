//! `bevy_strolle::StrollePlugin` for the H100 engine.
//!
//! Same shape as the reference plugin (`/bevy-strolle/src/lib.rs:29-84`, `stages.rs`, `rendering_node.rs`): the main world's meshes,
//! materials, images, instances, lights, sun and cameras are mirrored into the engine once per frame (extract in `ExtractSchedule`, apply
//! in `Render::Prepare`), and a render-graph node on the camera's view renders through the engine.  The CUDA engine composes into host
//! memory, so the node ends with one `write_texture` into the view's main texture where the reference records compute passes.
//!
//! `STROLLE_B200_DEVICES=0,1,2,3` selects the GPUs (default `0`); several devices = row strips of every camera's frame.
pub mod prelude {
    pub use crate::{StrolleCamera, StrollePlugin, StrolleSettings, StrolleSun};
}

mod sync;

use bevy::prelude::*;
use bevy::render::render_graph::{NodeRunError, RenderGraphApp, RenderGraphContext, ViewNode, ViewNodeRunner};
use bevy::render::renderer::{RenderContext, RenderQueue};
use bevy::render::view::ViewTarget;
use bevy::render::RenderApp;
pub use strolle as st;

/// Name of the render graph a camera selects with `CameraRenderGraph::new(bevy_strolle::graph::NAME)` (`/bevy-strolle/src/graph.rs`).
pub mod graph {
    pub const NAME: &str = "strolle";
    pub mod node {
        pub const RENDERING: &str = "strolle_rendering";
        pub const UPSCALING: &str = "strolle_upscaling";
    }
}

/// Per-camera settings (`/bevy-strolle/src/camera.rs`)
#[derive(Clone, Debug, Default, Component)]
pub struct StrolleCamera {
    pub mode: st::CameraMode,
}

/// The sun (`/bevy-strolle/src/sun.rs`)
#[derive(Clone, Debug, Default, Resource, Deref, DerefMut)]
pub struct StrolleSun {
    sun: st::Sun,
}

/// Engine-wide settings, read once when the plugin finishes building; insert the resource before `StrollePlugin` to change them.
/// `normal_maps`: shade with `StandardMaterial::normal_map_texture` and the mesh's `ATTRIBUTE_TANGENT` (off by default, as in the
/// reference, which ignores normal maps).
/// `bvh_refit_ticks`: up to this many frames in a row that only move entities refit the BVH on the GPU instead of rebuilding it
/// (0, the default, rebuilds every time, as the reference does).
/// `light_grid`: sample light candidates from a grid of the point lights that can reach each cell, this many cells along its
/// longest axis (1..=64; 0, the default, samples every light, as the reference does) - for scenes with many short-range lights.
/// `texture_filter`: filter material textures through mip chains (false, the default, takes the nearest texel, as the reference does).
/// `temporal_aa`: anti-alias with sub-pixel camera jitter and a temporal resolve (false, the default, renders one ray through each
/// pixel centre, as the reference does); needs one GPU.
/// `environment_map`: light the scene from an equirectangular HDR map in place of the procedural sky (None, the default, keeps the
/// reference's sky); put the sun (`StrolleSun`) below the horizon to light from the map alone.
/// `environment_map_sampling`: aim the GI bounce and sky draw at the environment map's bright texels (false, the default, draws
/// from the BRDF and the uniform hemisphere, as the reference does) - for HDRIs with a small, bright sun.
/// `tonemapping`: expose and tonemap the frame for display (`Tonemapping::None`, the default, clamps linear light, as the reference
/// does); with any other value the views receive `Rgba8UnormSrgb` frames instead of linear `Rgba32Float` ones.
/// `auto_exposure`: meter each camera's frame and adapt its exposure (false, the default, takes `exposure.ev`); needs one GPU.
/// `exposure`: the manual EV, the compensation and the metering's window, clamp and speeds.
/// `bloom`: a glow around light brighter than the display shows (None, the default, stores no glow); with `Some` the views receive
/// `Rgba8UnormSrgb` frames, with or without tonemapping; needs one GPU.
/// `depth_of_field`: defocus each camera's frames through a thin lens (None, the default, keeps them sharp); needs one GPU.
#[derive(Clone, Debug, Default, Resource)]
pub struct StrolleSettings {
    pub normal_maps: bool,
    pub bvh_refit_ticks: u32,
    pub light_grid: u32,
    pub texture_filter: bool,
    pub temporal_aa: bool,
    pub environment_map: Option<st::EnvironmentMap>,
    pub environment_map_sampling: bool,
    pub tonemapping: st::Tonemapping,
    pub auto_exposure: bool,
    pub exposure: st::Exposure,
    pub bloom: Option<st::Bloom>,
    pub depth_of_field: Option<st::DepthOfField>,
}

#[derive(Clone, Debug)]
pub struct EngineParams;

impl st::Params for EngineParams {
    type ImageHandle = AssetId<Image>;
    type InstanceHandle = Entity;
    type LightHandle = Entity;
    type MaterialHandle = AssetId<StandardMaterial>;
    type MeshHandle = AssetId<Mesh>;
}

#[derive(Resource, Deref, DerefMut)]
pub(crate) struct EngineResource(pub st::Engine<EngineParams>);

pub struct StrollePlugin;

impl Plugin for StrollePlugin {
    fn build(&self, app: &mut App) {
        app.insert_resource(StrolleSun::default());
        let Ok(render_app) = app.get_sub_app_mut(RenderApp) else { return };
        render_app.insert_resource(sync::Synced::default());
        sync::setup(render_app);
        render_app
            .add_render_sub_graph(graph::NAME)
            .add_render_graph_node::<ViewNodeRunner<RenderingNode>>(graph::NAME, graph::node::RENDERING)
            .add_render_graph_node::<ViewNodeRunner<bevy::core_pipeline::upscaling::UpscalingNode>>(graph::NAME, graph::node::UPSCALING)
            .add_render_graph_edges(graph::NAME, &[graph::node::RENDERING, graph::node::UPSCALING]);
    }

    fn finish(&self, app: &mut App) {
        let settings = app.world.get_resource::<StrolleSettings>().cloned().unwrap_or_default();
        let Ok(render_app) = app.get_sub_app_mut(RenderApp) else { return };
        let devices: Vec<i32> = std::env::var("STROLLE_B200_DEVICES")
            .ok()
            .map(|v| v.split(',').filter_map(|d| d.trim().parse().ok()).collect())
            .filter(|v: &Vec<i32>| !v.is_empty())
            .unwrap_or_else(|| vec![0]);
        let mut engine = st::Engine::new(&devices).expect("strolle_b200: no usable CUDA device (this engine has no CPU fallback)");
        engine.set_normal_maps(settings.normal_maps).expect("strolle_b200: ST_OPT_NORMAL_MAPS");
        engine.set_bvh_refit(settings.bvh_refit_ticks).expect("strolle_b200: ST_OPT_BVH_REFIT");
        engine.set_light_grid(settings.light_grid).expect("strolle_b200: ST_OPT_LIGHT_GRID");
        engine.set_texture_filter(settings.texture_filter).expect("strolle_b200: ST_OPT_TEXTURE_FILTER");
        engine.set_temporal_aa(settings.temporal_aa).expect("strolle_b200: ST_OPT_TEMPORAL_AA");
        engine.set_environment_map_sampling(settings.environment_map_sampling).expect("strolle_b200: ST_OPT_ENVIRONMENT_MAP_SAMPLING");
        engine.set_tonemapping(settings.tonemapping).expect("strolle_b200: ST_OPT_TONEMAPPING");
        engine.set_auto_exposure(settings.auto_exposure).expect("strolle_b200: ST_OPT_AUTO_EXPOSURE");
        engine.set_exposure(&settings.exposure).expect("strolle_b200: st_set_exposure");
        engine.set_bloom(settings.bloom.as_ref()).expect("strolle_b200: st_set_bloom");
        engine.set_depth_of_field(settings.depth_of_field.as_ref()).expect("strolle_b200: st_set_depth_of_field");
        sync::set_environment_map(&mut engine, settings.environment_map.as_ref());
        render_app.world.resource_mut::<sync::Synced>().tonemapped = settings.tonemapping != st::Tonemapping::None || settings.bloom.is_some();
        render_app.insert_resource(EngineResource(engine));
    }
}

/// `RenderingNode` (`/bevy-strolle/src/rendering_node.rs:14-36`)
#[derive(Default)]
pub(crate) struct RenderingNode;

impl ViewNode for RenderingNode {
    type ViewQuery = &'static ViewTarget;

    fn run(&self, graph: &mut RenderGraphContext, _render_context: &mut RenderContext, target: &ViewTarget, world: &World) -> Result<(), NodeRunError> {
        let entity = graph.view_entity();
        let engine = world.resource::<EngineResource>();
        let synced = world.resource::<sync::Synced>();
        let Some(camera) = synced.cameras.get(&entity) else { return Ok(()) };
        let mut frame = camera.frame.lock().unwrap();
        if let Err(err) = engine.render_camera(camera.handle, &mut frame) {
            error!("strolle: {err}");
            return Ok(());
        }
        let size = wgpu::Extent3d { width: frame.size.x, height: frame.size.y, depth_or_array_layers: 1 };
        let layout = wgpu::ImageDataLayout { offset: 0, bytes_per_row: Some(frame.size.x * frame.format.bytes_per_pixel() as u32), rows_per_image: Some(frame.size.y) };
        let copy = wgpu::ImageCopyTexture { texture: target.main_texture(), mip_level: 0, origin: wgpu::Origin3d { x: camera.position.x, y: camera.position.y, z: 0 }, aspect: wgpu::TextureAspect::All };
        world.resource::<RenderQueue>().write_texture(copy, &frame.pixels, layout, size);
        Ok(())
    }
}
