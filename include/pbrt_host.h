/*
 * pbrt_host.h -- C API of the C++ host mirror (librs_pbrt_b200.so) that sits ABOVE the GPU C ABI.
 *
 * rs_pbrt is compiled Rust and this image has no Rust toolchain, so the host side of the drop-in is
 * written in C++ and mirrors the reference's own call sequence for the path:
 *   pbrt_shape / pbrt_area_light_source      src/core/api.rs:2792-2870   -> pbrt_host_add_trianglemesh
 *   pbrt_look_at / make_camera               src/core/api.rs:486-514,1639-1689, src/cameras/perspective.rs:46-185,
 *                                            orthographic.rs:99-149, environment.rs:44-90
 *   pbrt_transform_times / animated camera   src/core/api.rs:497-502,2525-2529 -> pbrt_host_camera_motion
 *   make_film / make_filter                  src/core/film.rs:176-262, src/filters
 *   make_sampler ("sobol")                   src/samplers/sobol.rs:37-108
 *   make_integrator ("path")                 src/core/api.rs:285-321
 *   pbrt_cleanup: make_scene + render        src/core/api.rs:2352-2373
 *       BVHAccel::new                        src/accelerators/bvh.rs:96-392
 *       Scene::new                           src/core/scene.rs:27-51
 *       SamplerIntegrator::render            src/core/integrator.rs:70-220  (tile loop -> pbrt_gpu_render)
 *       Film::merge_film_tile / write_image  src/core/film.rs:346-371,437-528
 * All return 0 on success, negative PbrtStatus on error (pbrt_host_last_error()).
 */
#ifndef PBRT_HOST_H
#define PBRT_HOST_H
#include "pbrt_gpu.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct PbrtHost PbrtHost;

PbrtHost* pbrt_host_new(void);
void pbrt_host_free(PbrtHost* h);
const char* pbrt_host_last_error(void);

/* Material "<kind>" with constant textures; returns the material index (>= 0). */
int pbrt_host_add_material(PbrtHost* h, uint32_t kind, const float params[24]);
/* Material "mix" (api.rs:678-705, src/materials/mixmat.rs): m1 / m2 = indices of "namedmaterial1" / "namedmaterial2" as returned by earlier
 * calls, amount = the constant "amount" spectrum (default 0.5).  Returns the material index (>= 0). */
int pbrt_host_add_material_mix(PbrtHost* h, int m1, int m2, const float amount[3]);
/* Texture "name" "spectrum" | "float" "imagemap" (api.rs make_texture -> ImageTexture::new, imagemap.rs:35-97): rgb = the decoded image,
 * width x height RGB in [0,1], row 0 = TOP of the image as the decoder delivers it.  This call does what ImageTexture::new does
 * before MipMap::new: the y flip and convert_in (inverse sRGB gamma when `gamma` -- the reference's default for .png/.tga --, then
 * * scale) and, for a float texture (float_valued != 0), convert_to_float = the luminance y() of the result (imagemap.rs:155-157).
 * wrap: PbrtWrap.  Returns the texture index (>= 0). */
int pbrt_host_add_texture_image(PbrtHost* h, const float* rgb, uint32_t width, uint32_t height, int float_valued, int trilinear, float max_anisotropy,
                                uint32_t wrap, float scale, int gamma, float uscale, float vscale, float udelta, float vdelta);
/* Texture "constant" (value[0] alone for a float texture), "scale" (tex1 * tex2) and "mix" (tex1 * (1 - amount) + tex2 * amount;
 * amount is a float texture): operands are indices returned by earlier pbrt_host_add_texture_* calls. */
int pbrt_host_add_texture_constant(PbrtHost* h, const float value[3], int float_valued);
int pbrt_host_add_texture_scale(PbrtHost* h, int tex1, int tex2);
int pbrt_host_add_texture_mix(PbrtHost* h, int tex1, int tex2, int amount);
/* Bind texture `texture` to parameter group `group` of `material` (the group table in pbrt_gpu.h: matte {Kd | sigma},
 * plastic {Kd, Ks | roughness}, ...), as `"texture Kd" "name"` does in the scene file. */
int pbrt_host_material_texture(PbrtHost* h, int material, int group, int texture);
/* "mapping" of an image texture other than "uv": PBRT_MAP_SPHERICAL / PBRT_MAP_CYLINDRICAL with m = world_to_texture (16 floats,
 * row-major), PBRT_MAP_PLANAR with m = {v1[3], v2[3]} (udelta / vdelta of the image call are its offsets) */
int pbrt_host_texture_mapping(PbrtHost* h, int texture, uint32_t mapping, const float* m);
/* "texture bumpmap": a float texture that perturbs the material's shading frame (Material::bump, material.rs:116-219) */
int pbrt_host_material_bump(PbrtHost* h, int material, int texture);
/* Shape "trianglemesh" with WORLD-space vertices.  material < 0 = Material "none".  emit_L != NULL puts an
 * AreaLightSource "diffuse" in scope: every triangle becomes its own DiffuseAreaLight (api.rs:2810-2852).
 * Returns the mesh index. */
int pbrt_host_add_trianglemesh(PbrtHost* h, uint32_t n_tris, const uint32_t* indices, uint32_t n_verts, const float* P, const float* N,
                               const float* S, const float* UV, int reverse_orientation, int swaps_handedness, int material,
                               const float* emit_L, int two_sided);
/* "texture alpha" / "texture shadowalpha" of the Shape (api.rs:1920-1964): float textures returned by pbrt_host_add_texture_* (a
 * constant 0 for `"float alpha" 0`), -1 = none.  `mesh` is the index pbrt_host_add_trianglemesh returned. */
int pbrt_host_mesh_alpha(PbrtHost* h, int mesh, int alpha_texture, int shadow_alpha_texture);
/* ObjectBegin / ObjectEnd / ObjectInstance (src/core/api.rs:3001-3109).  Meshes added between begin and end belong to the object
 * (no emitters: the reference rejects area lights in objects) and are only reachable through its instances.  instance_to_world:
 * the CTM at the ObjectInstance directive, row-major 4x4, NULL = identity.  pbrt_host_instancing selects PbrtInstancing. */
int pbrt_host_object_begin(PbrtHost* h); /* returns the object id */
int pbrt_host_object_end(PbrtHost* h);
int pbrt_host_object_instance(PbrtHost* h, int object, const float* instance_to_world);
int pbrt_host_instancing(PbrtHost* h, uint32_t mode);
/* LightSource "point" / "spot" / "distant" (make_light, src/core/api.rs:769-925) with the identity CTM of a world block.
 * `scale` may be NULL (= 1).  Lights keep their declaration order relative to the emissive meshes (scene.lights order). */
int pbrt_host_add_light_point(PbrtHost* h, const float from[3], const float I[3], const float scale[3]);
int pbrt_host_add_light_spot(PbrtHost* h, const float from[3], const float to[3], const float I[3], const float scale[3], float coneangle,
                             float conedeltaangle);
int pbrt_host_add_light_distant(PbrtHost* h, const float from[3], const float to[3], const float L[3], const float scale[3]);
/* LightSource "infinite": texels = NULL for a constant light (InfiniteAreaLight::default, infinite.rs:250-300), else a
 * width x height RGB lat-long map (any resolution) that is multiplied by L*scale as the reference does on load.
 * light_to_world / world_to_light: row-major 3x3 rotations of the CTM and its inverse, both NULL for identity. */
/* LightSource "goniometric" / "projection" under the current transform: light_to_world / world_to_light are the CTM and its inverse
 * (row-major 4x4), texels an RGB map of width x height with row 0 first as the .hdr file stores it (NULL: no "mapname"; required for
 * a projection light), fov in degrees (the reference's default is 45). */
int pbrt_host_add_light_goniometric(PbrtHost* h, const float I[3], const float scale[3], const float* texels, uint32_t width, uint32_t height,
                                    const float light_to_world[16], const float world_to_light[16]);
int pbrt_host_add_light_projection(PbrtHost* h, const float I[3], const float scale[3], const float* texels, uint32_t width, uint32_t height, float fov,
                                   const float light_to_world[16], const float world_to_light[16]);
int pbrt_host_add_light_infinite(PbrtHost* h, const float L[3], const float scale[3], const float* texels, uint32_t width, uint32_t height,
                                 const float* light_to_world, const float* world_to_light);
int pbrt_host_look_at(PbrtHost* h, const float eye[3], const float look[3], const float up[3]);
/* TransformTimes start end (api.rs:2525-2529; defaults 0 and 1): the times of the start and end keyframes of every AnimatedTransform. */
int pbrt_host_transform_times(PbrtHost* h, float start, float end);
/* The camera's end keyframe (`ActiveTransform EndTime` before the Camera directive): camera_to_world at the end time, row-major 4x4;
 * the start keyframe is the one pbrt_host_look_at set.  NULL = a static camera again.  make_camera then builds the camera's
 * AnimatedTransform (api.rs:497-502); pbrt_host_motion_desc hands it to pbrt_gpu_scene_create_motion. */
int pbrt_host_camera_motion(PbrtHost* h, const float* camera_to_world_end);
/* Film "image": crop = {x0,x1,y0,y1} in [0,1] or NULL; filter_name "box" | "gaussian" | "triangle" (xwidth/ywidth = radius) */
int pbrt_host_film(PbrtHost* h, int xres, int yres, const float* crop, const char* filter_name, float xwidth, float ywidth, float filter_alpha,
                   float max_sample_luminance);
/* Camera "perspective"; screen_window = {xmin,xmax,ymin,ymax} or NULL (derived from the frame aspect ratio). Call after pbrt_host_film. */
int pbrt_host_camera_perspective(PbrtHost* h, float fov, float lens_radius, float focal_distance, float shutter_open, float shutter_close,
                                 const float* screen_window);
/* Camera "orthographic" (OrthographicCamera::create, src/cameras/orthographic.rs:99-149): raster_to_camera from
 * Transform::orthographic(0, 1), the screen window (NULL: from the frame aspect ratio) and the film's full resolution.  The
 * reference's defaults are lensradius 0 and focaldistance 1e6. */
int pbrt_host_camera_orthographic(PbrtHost* h, float lens_radius, float focal_distance, float shutter_open, float shutter_close,
                                  const float* screen_window);
/* Camera "environment" (EnvironmentCamera::create, src/cameras/environment.rs:44-90): camera_to_world, the shutter and the film's
 * full resolution; it reads no screen window and no lens.  Call after pbrt_host_film. */
int pbrt_host_camera_environment(PbrtHost* h, float shutter_open, float shutter_close);
/* Film "diagonal" in millimetres (film.rs:250, default 35): the realistic camera's film size.  Call before the camera. */
int pbrt_host_film_diagonal(PbrtHost* h, float mm);
/* Camera "realistic" (RealisticCamera::create / new, src/cameras/realistic.rs:50-197): lens_mm holds the lens file's n_values
 * numbers, rows {radius, thickness, eta, diameter} in mm.  The stop's diameter is replaced by aperture_diameter unless that is
 * larger; the last thickness is set by focus_thick_lens; the 64 exit-pupil bins are bounded on host threads.  focus_binary_search
 * is not restated: the reference discards its result.  Where the reference asserts or panics (no ray through the thick-lens
 * approximation, a focus distance too short) and for a row count that is not a positive multiple of four: PBRT_E_INVALID.
 * Call after pbrt_host_film (and pbrt_host_film_diagonal). */
int pbrt_host_camera_realistic(PbrtHost* h, const float* lens_mm, int n_values, float aperture_diameter, float focus_distance, int simple_weighting,
                               float shutter_open, float shutter_close);
int pbrt_host_sampler_sobol(PbrtHost* h, int pixel_samples);
/* Sampler "halton" (src/samplers/halton.rs:162-172), the reference's default sampler; any pixel_samples >= 1. */
int pbrt_host_sampler_halton(PbrtHost* h, int pixel_samples, int sample_at_pixel_center);
/* Integrator "path"; pixel_bounds = {x0,x1,y0,y1} or NULL */
/* Integrator "ao" (CreateAOIntegrator, src/core/api.rs:411-435): nsamples (64), cossample (true) */
int pbrt_host_integrator_ao(PbrtHost* h, int n_samples, int cos_sample);
/* Integrator "directlighting": maxdepth (5), strategy PbrtDirectStrategy ("all" | "one"); Integrator "whitted": maxdepth (5) */
int pbrt_host_integrator_direct(PbrtHost* h, uint32_t max_depth, uint32_t strategy, const int32_t* pixel_bounds);
int pbrt_host_integrator_whitted(PbrtHost* h, uint32_t max_depth, const int32_t* pixel_bounds);
/* "nsamples" of the LightSource / AreaLightSource statements that follow (default 1) */
int pbrt_host_light_samples(PbrtHost* h, uint32_t n_samples);
int pbrt_host_integrator_path(PbrtHost* h, uint32_t max_depth, float rr_threshold, uint32_t light_strategy, const int32_t* pixel_bounds);
/* WorldEnd up to (not including) render: builds the BVH, the light list and the flat description. */
int pbrt_host_world_end(PbrtHost* h, uint32_t max_prims_in_node, int n_threads);

const PbrtSceneDesc* pbrt_host_scene_desc(const PbrtHost* h);
const PbrtRenderParams* pbrt_host_render_params(const PbrtHost* h);
/* The motion description of the built scene, NULL when nothing in it is animated. */
const PbrtMotionDesc* pbrt_host_motion_desc(const PbrtHost* h);
/* The camera model of the built scene (its kind and Film.full_resolution) for pbrt_gpu_scene_create_camera. */
const PbrtCameraModel* pbrt_host_camera_model(const PbrtHost* h);
/* RealisticCamera::bound_exit_pupil of the 64 film-radius bins (realistic.rs:100-139,573-652) for a lens given in metres, film
 * side last, whose last thickness is already the lens-film distance: 64 x {pmin.x, pmin.y, pmax.x, pmax.y}.  What
 * pbrt_host_camera_realistic computes after focusing. */
int pbrt_host_lens_exit_pupil(const PbrtLensElement* elements, int n_elements, float film_diagonal_m, float* bounds);
/* The realistic camera of the built scene for pbrt_gpu_scene_create_lens; NULL for any other camera. */
const PbrtRealisticLens* pbrt_host_lens(const PbrtHost* h);

/* Integrator::render(scene, num_threads): uploads the scene, renders pixel_rect (NULL = whole sample bounds) on `device`
 * through pbrt_gpu_render, and merges the result into the Film like merge_film_tile. */
int pbrt_host_render(PbrtHost* h, int device, const int32_t* pixel_rect, PbrtStats* stats);
/* Film access: raw {contrib_sum rgb, filter_weight_sum} (area*4), and Film::write_image's float RGB (area*3). */
const float* pbrt_host_film_rgbw(const PbrtHost* h);
int pbrt_host_film_clear(PbrtHost* h);
int pbrt_host_film_add_rgbw(PbrtHost* h, const float* rgbw); /* merge an externally rendered film (e.g. the NCCL-reduced one) */
int pbrt_host_film_rgb(const PbrtHost* h, float* rgb_out);
/* Film::write_image: 8-bit sRGB; writes a binary PPM (the reference writes the same bytes as pbrt.png) */
int pbrt_host_write_image(const PbrtHost* h, const char* path);

/* BVHAccel::new on bare bounds (n*6 floats).  nodes_out holds 2n entries, ordered_out n entries. */
int pbrt_host_bvh_build(const float* bounds, uint32_t n, uint32_t max_prims_in_node, int n_threads, PbrtBvhNode* nodes_out,
                        uint32_t* n_nodes_out, uint32_t* ordered_out);

#ifdef __cplusplus
}
#endif
#endif
