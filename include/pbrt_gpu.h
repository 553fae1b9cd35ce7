/*
 * pbrt_gpu.h -- C ABI of the H100 PathIntegrator hot path (librs_pbrt_b200.so).
 *
 * This is the drop-in boundary for rs_pbrt's SamplerIntegrator::render tile
 * loop.  The reference has no FFI of its own; the Rust-internal call that is
 * replaced is
 *     Integrator::render(&mut self, scene: &Scene, num_threads: u8)
 *         src/core/integrator.rs:39-46,70   (tile loop :86-218)
 * and the two scene queries the loop bottoms out in,
 *     Scene::intersect / Scene::intersect_p            src/core/scene.rs:55,67
 *
 * Everything here is plain C: pointers to caller-owned HOST memory unless a
 * parameter is explicitly named d_* (device).  The library copies what it
 * needs at pbrt_gpu_scene_create(); there are no callbacks.  A handle may be
 * used from one thread at a time.  Every function returns 0 on success and a
 * negative PbrtStatus otherwise; PBRT_E_UNSUPPORTED tells the caller to fall
 * back to its own CPU loop (the library itself has NO CPU fallback).
 *
 * INTEGRATION.md shows the Rust `extern "C"` block that binds these.
 *
 * ABI versions (pbrt_gpu_abi_version): 1 = area lights, Sobol', path integrator; 2 = all light kinds, Halton, ao, object instances;
 * 3 = image textures (PbrtTexture, PbrtMaterial.tex / bump, PbrtSceneDesc.textures), PbrtLight.n_samples, the directlighting and
 * whitted integrators (PbrtRenderParams.direct_strategy); 4 = PbrtStats.shade_slots / shaded_vertices, tile-interleaved rendering
 * (pbrt_gpu_render_tiles*) and the one-process multi-device render (pbrt_gpu_render_multi); within 4, the animated camera
 * (pbrt_gpu_scene_create_motion and its new structs: nothing that existed changed); within 4, goniometric and projection lights
 * (PBRT_LIGHT_GONIOMETRIC / PROJECTION and PbrtLight.fov in the former pad word); within 4, pbrt_gpu_scene_create_multi; within 4,
 * orthographic and environment cameras (pbrt_gpu_scene_create_camera, PbrtCameraModel); within 4, the realistic camera
 * (pbrt_gpu_scene_create_lens, PbrtRealisticLens, PBRT_CAMERA_REALISTIC).  Structs only ever grow at their end
 * within a version step, and a zero-initialised new field means "as before".
 */
#ifndef PBRT_GPU_H
#define PBRT_GPU_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PBRT_GPU_ABI_VERSION 4

typedef enum PbrtStatus {
    PBRT_OK = 0,
    PBRT_E_INVALID = -1,     /* malformed description (null pointer, index out of range, ...) */
    PBRT_E_UNSUPPORTED = -2, /* feature outside the GPU path: caller runs its CPU loop */
    PBRT_E_CUDA = -3,        /* CUDA runtime error; pbrt_gpu_last_error() has the text */
    PBRT_E_NO_DEVICE = -4    /* no usable sm_90 (H100) device */
} PbrtStatus;

/* == LinearBVHNode, 32 bytes (src/accelerators/bvh.rs:77-85).
 * interior: offset = index of second child (first child is self+1), n_prims = 0, axis = split axis
 * leaf:     offset = first primitive in PbrtSceneDesc.tris, n_prims > 0 */
typedef struct PbrtBvhNode {
    float pmin[3];
    float pmax[3];
    int32_t offset;
    uint16_t n_prims;
    uint8_t axis;
    uint8_t pad;
} PbrtBvhNode;

/* One GeometricPrimitive{Triangle}, listed in BVHAccel.primitives order
 * (src/accelerators/bvh.rs:91, src/core/primitive.rs:100-105, src/shapes/triangle.rs:84-87). */
#define PBRT_NO_MATERIAL 0xffffffffu
#define PBRT_MESH_INSTANCE 0xffffffffu /* PbrtTri.mesh: this primitive is a TransformedPrimitive; v[0] = index into PbrtSceneDesc.instances */
typedef struct PbrtTri {
    uint32_t v[3];      /* vertex indices into the mesh's arrays (TriangleMesh.vertex_indices[3*id..]) */
    uint32_t mesh;      /* index into PbrtSceneDesc.meshes */
    uint32_t material;  /* index into PbrtSceneDesc.materials, or PBRT_NO_MATERIAL (Material "none") */
    int32_t area_light; /* index into PbrtSceneDesc.lights of this primitive's DiffuseAreaLight, or -1 */
} PbrtTri;

/* TriangleMesh in WORLD space (src/shapes/triangle.rs:24-46; api.rs:1891-1971 transforms at load). */
typedef struct PbrtMesh {
    const float* p;  /* 3*n_verts, required */
    const float* n;  /* 3*n_verts or NULL */
    const float* s;  /* 3*n_verts or NULL */
    const float* uv; /* 2*n_verts or NULL */
    uint32_t n_verts;
    uint8_t reverse_orientation;
    uint8_t transform_swaps_handedness;
    uint8_t pad[2];
    /* ABI v4: TriangleMesh.alpha_mask / shadow_alpha_mask (triangle.rs:39-40; "alpha" / "shadowalpha" of the Shape, api.rs:1920-1964):
     * 0 = none, else 1 + index of a FLOAT texture in PbrtSceneDesc.textures (a constant 0 for `"float alpha" 0`).  A candidate hit whose
     * mask evaluates to exactly 0 at the hit's (p, uv) is rejected: Triangle::intersect tests alpha_mask only (triangle.rs:313-330),
     * Triangle::intersect_p both (triangle.rs:593-654).  Emissive meshes with a mask are PBRT_E_UNSUPPORTED (pdf_li's single-triangle
     * test would have to evaluate it too). */
    uint32_t alpha;
    uint32_t shadow_alpha;
} PbrtMesh;

/* Materials with constant textures pre-evaluated by the caller
 * (src/textures/constant.rs:17-20).  params layout per kind:
 *   MATTE     Kd[0..3) sigma[3]                                         materials/matte.rs:43-86
 *   PLASTIC   Kd[0..3) Ks[3..6) roughness[6] remap[7]                   materials/plastic.rs:57-125
 *   METAL     eta[0..3) k[3..6) urough[6] vrough[7] remap[8]            materials/metal.rs:144-205
 *   MIRROR    Kr[0..3)                                                  materials/mirror.rs:34-70
 *   GLASS     Kr[0..3) Kt[3..6) index[6] urough[7] vrough[8] remap[9]   materials/glass.rs:83-211
 *   UBER      Kd[0..3) Ks[3..6) Kr[6..9) Kt[9..12) opacity[12..15)
 *             urough[15] vrough[16] eta[17] remap[18]                   materials/uber.rs:114-259
 *   SUBSTRATE Kd[0..3) Ks[3..6) urough[6] vrough[7] remap[8]            materials/substrate.rs:62-114
 *   TRANSLUCENT Kd[0..3) Ks[3..6) reflect[6..9) transmit[9..12)
 *             roughness[12] remap[13]                                   materials/translucent.rs:48-189
 *   MIX       amount[0..3) m1[3] m2[4]                                   materials/mixmat.rs:29-98
 * (remap = 1.0f when "remaproughness" is true.)  Anything else => PBRT_E_UNSUPPORTED.
 * MIX (MixMaterial, api.rs:678-705): m1 / m2 are the indices of "namedmaterial1" / "namedmaterial2" in PbrtSceneDesc.materials,
 * stored as floats (exact below 2^24), each LOWER than the mix's own index (a named material exists before the mix that names it).
 * Its lobe list is m1's lobes scaled by s1 = clamp(amount) followed by m2's scaled by s2 = clamp(1 - s1) (every BxDF's sc_opt,
 * reflection.rs:714 ff.); eta and the shading frame are m1's.  A child that is itself a MIX ignores the scale handed down to it, as
 * the reference's does (mixmat.rs:48 `_scale`).  In this version the amount is a constant, the children carry no textures and no bump
 * map, and the lobes of both children together number at most five (the reference allows eight): otherwise PBRT_E_UNSUPPORTED. */
typedef enum PbrtMaterialKind {
    PBRT_MAT_MATTE = 0,
    PBRT_MAT_PLASTIC = 1,
    PBRT_MAT_METAL = 2,
    PBRT_MAT_MIRROR = 3,
    PBRT_MAT_GLASS = 4,
    PBRT_MAT_UBER = 5,
    PBRT_MAT_SUBSTRATE = 6,
    PBRT_MAT_TRANSLUCENT = 7, /* ABI v4, round 2: Lambertian reflection + transmission, microfacet reflection + transmission (eta 1.5) */
    PBRT_MAT_MIX = 8          /* ABI v4, round 2: MixMaterial over two earlier materials */
} PbrtMaterialKind;

/* Image textures (ABI v3).  A parameter of a material may be bound to an ImageTexture (src/textures/imagemap.rs:17-150) with a
 * UVMapping2D (src/core/texture.rs:93-122): PbrtMaterial.tex[g] = 1 + index into PbrtSceneDesc.textures for parameter group g,
 * 0 = the constant in params[].  Groups, in the order of the layout table above (spectrum-valued ones first, then the floats):
 *   MATTE {Kd | sigma}  PLASTIC {Kd, Ks | roughness}  METAL {eta, k | urough, vrough}  MIRROR {Kr}
 *   GLASS {Kr, Kt | index, urough, vrough}  UBER {Kd, Ks, Kr, Kt, opacity | urough, vrough, eta}  SUBSTRATE {Kd, Ks | urough, vrough}
 *   TRANSLUCENT {Kd, Ks, reflect, transmit | roughness}  MIX {amount} (validated, then PBRT_E_UNSUPPORTED: see above)
 * A spectrum group takes an ImageTexture<Spectrum> (channels = 3), a float group an ImageTexture<Float> (channels = 1: the texels
 * after convert_to_float, imagemap.rs:155-157).  pbrt_material_tex_offset() below gives the params[] offset of a group.
 * The texture is evaluated at every shaded hit as Material::compute_scattering_functions does (e.g. matte.rs:61-69), after
 * SurfaceInteraction::compute_differentials (interaction.rs:388-474): camera rays carry PerspectiveCamera's ray differentials
 * (perspective.rs:190-280, scaled by 1/sqrt(spp), integrator.rs:140-144), every later ray of a path has none (interaction.rs:493-503),
 * so its lookups are level-0 bilinear.  MipMap::lookup (mipmap.rs:233-296) is trilinear or EWA as `trilinear` says. */
#define PBRT_MAX_TEX_GROUPS 8
typedef enum PbrtWrap { PBRT_WRAP_REPEAT = 0, PBRT_WRAP_BLACK = 1, PBRT_WRAP_CLAMP = 2 } PbrtWrap;
/* Texture kinds: an image (the fields below), a ConstantTexture (src/textures/constant.rs; value[]), a ScaleTexture
 * (src/textures/scale.rs: tex1 * tex2) or a MixTexture (src/textures/mix.rs: tex1 * (1 - amount) + tex2 * amount).  child[] = 1 + index
 * of tex1, tex2, amount, each LOWER than the node's own index (a DAG in creation order, at most PBRT_MAX_TEXTURE_DEPTH levels);
 * children have the node's `channels`, amount has 1. */
typedef enum PbrtTextureMapping { PBRT_MAP_UV = 0, PBRT_MAP_SPHERICAL = 1, PBRT_MAP_CYLINDRICAL = 2, PBRT_MAP_PLANAR = 3 } PbrtTextureMapping;
typedef enum PbrtTextureKind { PBRT_TEX_IMAGE = 0, PBRT_TEX_CONSTANT = 1, PBRT_TEX_SCALE = 2, PBRT_TEX_MIX = 3 } PbrtTextureKind;
#define PBRT_MAX_TEXTURE_DEPTH 4
typedef struct PbrtTexture {
    uint32_t res[2];      /* width, height of `texels` (any size; not a power of two => MipMap::new's Lanczos zoom, mipmap.rs:60-150) */
    const float* texels;  /* channels*res[0]*res[1] values, row 0 at t = 0, as handed to MipMap::new: after the y flip and convert_in (gamma, scale; imagemap.rs:62-84) */
    uint32_t channels;    /* 3 = ImageTexture<Spectrum> (RGB), 1 = ImageTexture<Float> */
    uint32_t trilinear;   /* "trilinear" parameter (do_trilinear) */
    float max_anisotropy; /* "maxanisotropy", default 8 */
    uint32_t wrap;        /* PbrtWrap ("wrap": repeat | black | clamp) */
    float su, sv, du, dv; /* UVMapping2D: "uscale" "vscale" "udelta" "vdelta" */
    uint32_t mapping;     /* PbrtTextureMapping of an image (0 = UVMapping2D with su, sv, du, dv) */
    float map_m[16];      /* SPHERICAL / CYLINDRICAL: world_to_texture, row-major 4x4 (texture.rs:123-215);
                             PLANAR: vs = map_m[0..3), vt = map_m[3..6), and ds, dt in du, dv (texture.rs:217-252) */
    uint32_t kind;        /* PbrtTextureKind (0 = image: the zero-initialised default) */
    float value[3];       /* CONSTANT (value[0] for channels == 1) */
    uint32_t child[3];    /* SCALE: tex1, tex2; MIX: tex1, tex2, amount */
} PbrtTexture;

typedef struct PbrtMaterial {
    uint32_t kind;
    float params[24];
    uint32_t tex[PBRT_MAX_TEX_GROUPS]; /* 0 = constant, else 1 + texture index (see above) */
    uint32_t bump;  /* "bumpmap": 0 = none, else 1 + index of a float texture (channels == 1); Material::bump (src/core/material.rs:116-219)
                       perturbs the shading frame before the other textures are evaluated */
} PbrtMaterial;
/* params[] offset of parameter group g of a material kind, -1 = no such group; *n_values = 3 (spectrum) or 1 (float) */
static inline int pbrt_material_tex_offset(uint32_t kind, int g, int* n_values) {
    static const signed char off[9][PBRT_MAX_TEX_GROUPS] = {{0, 3, -1, -1, -1, -1, -1, -1}, {0, 3, 6, -1, -1, -1, -1, -1}, {0, 3, 6, 7, -1, -1, -1, -1},
                                                             {0, -1, -1, -1, -1, -1, -1, -1}, {0, 3, 6, 7, 8, -1, -1, -1}, {0, 3, 6, 9, 12, 15, 16, 17},
                                                             {0, 3, 6, 7, -1, -1, -1, -1}, {0, 3, 6, 9, 12, -1, -1, -1},
                                                             {0, -1, -1, -1, -1, -1, -1, -1}};
    static const signed char n_spectrum[9] = {1, 2, 2, 1, 2, 5, 2, 4, 1};
    if (kind > 8u || g < 0 || g >= PBRT_MAX_TEX_GROUPS || off[kind][g] < 0) return -1;
    if (n_values) *n_values = g < n_spectrum[kind] ? 3 : 1;
    return off[kind][g];
}

/* One TransformedPrimitive (src/core/primitive.rs:198-272) = one ObjectInstance of an object that was defined between ObjectBegin /
 * ObjectEnd (src/core/api.rs:3001-3109).  The object's primitives have their own BVHAccel (api.rs:3050-3080): its nodes are a block of
 * PbrtSceneDesc.nodes starting at `root`, with ABSOLUTE child / primitive offsets; its triangles sit in PbrtSceneDesc.tris like any
 * other (they may not be instances themselves, nor area lights).  m / m_inv are instance_to_world as the reference carries them
 * (Transform.m, Transform.m_inv); rays enter the object through m_inv (Transform::transform_ray with its error offset,
 * transform.rs:538-594), interactions leave through m (transform_surface_interaction, transform.rs:815-860). */
typedef struct PbrtInstance {
    uint32_t root;
    uint32_t identity; /* Transform::is_identity() (transform.rs:291-308): selects the reference's identity-instance behaviour */
    float m[16];
    float m_inv[16];
} PbrtInstance;

/* How an instance hit is reported (SURVEY quirk Q7).  REFERENCE restates TransformedPrimitive::intersect as written: an instance
 * with an identity transform shortens the ray (and overwrites the interaction) but reports NO hit, any other instance reports the
 * hit but transform_surface_interaction clears `primitive` (transform.rs:856), so the surface has no material and no emission and
 * PathIntegrator walks through it (path.rs:109-116) -- while shadow rays are blocked by it.  FIXED is pbrt-v3's behaviour: the hit
 * keeps its primitive (material), identity or not. */
typedef enum PbrtInstancing { PBRT_INSTANCING_REFERENCE = 0, PBRT_INSTANCING_FIXED = 1 } PbrtInstancing;

/* scene.lights in declaration order (src/core/scene.rs:20,37-44).
 *   DIFFUSE_AREA  DiffuseAreaLight over one triangle (src/lights/diffuse.rs:19-24; one light per emissive
 *                 triangle, api.rs:2810-2852): L = l_emit, tri, two_sided, area
 *   POINT         PointLight   (src/lights/point.rs):   L = I (intensity), p = p_light
 *   SPOT          SpotLight    (src/lights/spot.rs):    L = I, p = p_light, w2l = upper 3x3 of world_to_light,
 *                 cos_total_width, cos_falloff_start
 *   DISTANT       DistantLight (src/lights/distant.rs): L = radiance, p = w_light (normalised, world space); the
 *                 world radius of DistantLight::preprocess is derived from world_bound by the library
 *   INFINITE      InfiniteAreaLight (src/lights/infinite.rs): env_texels = the lat-long radiance map the reference hands to
 *                 MipMap::new (RGB f32, row-major, already multiplied by L*scale; env_res = {1,1} and one texel for a light
 *                 without "mapname", infinite.rs:250-300), l2w / w2l = light_to_world / world_to_light rotations.  The library
 *                 restates InfiniteAreaLight::new: a map whose resolution is not a power of two is resampled to the next one
 *                 (MipMap::new's 4-tap Lanczos zoom, mipmap.rs:60-150), then the MIP pyramid (power()), the 2w x 2h
 *                 Distribution2D (sampling.rs:150-198) and the world radius are derived.
 *   GONIOMETRIC   GonioPhotometricLight (src/lights/goniometric.rs): L = I * scale, p = p_light, w2l = upper 3x3 of world_to_light,
 *                 env_res / env_texels = the map exactly as new_hdr hands it to MipMap::new (RGB f32, row 0 = the file's first row: the
 *                 constructor does not flip rows).  env_texels == NULL means no "mapname": scale(w) is exactly 1.  The radiance toward
 *                 a point is L * lookup(phi / 2pi, theta / pi) / d^2 of the light-space direction normalize(w2l * w) with y and z
 *                 swapped (goniometric.rs:233-265).
 *   PROJECTION    ProjectionLight (src/lights/projection.rs): L, p, w2l and the map as for GONIOMETRIC, fov = "fov" (default 45).
 *                 The library restates the constructor (screen window from the map's aspect, Transform::perspective(fov, 1e-3,
 *                 1e30), cos_total_width) and projection(w) (:339-360).  env_texels is required (NULL is PBRT_E_INVALID): a projection
 *                 light without "mapname" is black in the reference (I = 0, at the origin), and the caller hands it over as a
 *                 POINT light with L = 0 and p = 0, which gives the same samples, ray counts and power.
 *   Both: a map larger than 16384 texels on a side is PBRT_E_UNSUPPORTED; a zero resolution with texels, or a p / w2l / fov that is
 *   not finite (fov outside (0, 180) for PROJECTION) is PBRT_E_INVALID.  Not allowed inside object instances (neither is the reference).
 * Delta lights take the `is_delta_light` branch of estimate_direct (integrator.rs:470-480: no MIS, no BSDF sample). Rays that
 * leave the scene collect Le of every infinite light (path.rs:267-275, integrator.rs:560-562). */
typedef enum PbrtLightKind {
    PBRT_LIGHT_DIFFUSE_AREA = 0, PBRT_LIGHT_POINT = 1, PBRT_LIGHT_SPOT = 2, PBRT_LIGHT_DISTANT = 3, PBRT_LIGHT_INFINITE = 4,
    PBRT_LIGHT_GONIOMETRIC = 5, PBRT_LIGHT_PROJECTION = 6 /* ABI v4 */
} PbrtLightKind;
#define PBRT_MAX_INFINITE_LIGHTS 4
typedef struct PbrtLight {
    uint32_t kind;
    float L[3];        /* l_emit | I | L */
    uint32_t tri;      /* area: index into PbrtSceneDesc.tris of the emitting triangle */
    uint32_t two_sided;
    float area;        /* area: DiffuseAreaLight.area == Triangle::area() at creation */
    float p[3];        /* point/spot: p_light; distant: w_light */
    float w2l[9];      /* spot, infinite, goniometric, projection: upper 3x3 of world_to_light, row-major */
    float cos_total_width, cos_falloff_start; /* spot */
    float l2w[9];      /* infinite: light_to_world rotation, row-major */
    uint32_t env_res[2];      /* infinite, goniometric, projection: map resolution {width, height} */
    const float* env_texels;  /* infinite, goniometric, projection: env_res[0] * env_res[1] RGB texels */
    uint32_t n_samples;       /* "nsamples"/"samples" of the light (Light::get_n_samples; 0 reads as 1): DirectLightingIntegrator "all" */
    float fov;                /* projection: "fov" in degrees (was a zero pad word: the layout is unchanged) */
} PbrtLight;

/* PerspectiveCamera (src/cameras/perspective.rs:23-43); row-major 4x4, m[r][c] = a[4*r+c].
 * camera_to_world is the camera's start transform; an animated camera also hands its AnimatedTransform to
 * pbrt_gpu_scene_create_motion (below). */
typedef struct PbrtCamera {
    float raster_to_camera[16];
    float camera_to_world[16];
    float lens_radius;
    float focal_distance;
    float shutter_open;
    float shutter_close;
} PbrtCamera;

typedef struct PbrtSceneDesc {
    const PbrtBvhNode* nodes;
    uint32_t n_nodes;
    const PbrtTri* tris;
    uint32_t n_tris;
    const PbrtMesh* meshes;
    uint32_t n_meshes;
    const PbrtMaterial* materials;
    uint32_t n_materials;
    const PbrtLight* lights;
    uint32_t n_lights;
    PbrtCamera camera;
    float world_bound[6]; /* Scene.world_bound pmin,pmax (scene.rs:23) -- spatial light grid */
    const struct PbrtInstance* instances; /* object instances referenced by PbrtTri entries with mesh == PBRT_MESH_INSTANCE */
    uint32_t n_instances;
    const PbrtTexture* textures; /* image textures referenced by PbrtMaterial.tex (ABI v3) */
    uint32_t n_textures;
} PbrtSceneDesc;

typedef enum PbrtLightStrategy {
    PBRT_LIGHTS_UNIFORM = 0,
    PBRT_LIGHTS_POWER = 1,
    PBRT_LIGHTS_SPATIAL = 2 /* default; a single light always degrades to UNIFORM (lightdistrib.rs:397) */
} PbrtLightStrategy;

/* The two GlobalSamplers of the reference: Sampler "sobol" (src/samplers/sobol.rs) and the crate default Sampler "halton"
 * (src/samplers/halton.rs: base-2/3 pixel strata of at most 128 x 243, dimensions >= 2 through the radical-inverse digit
 * permutations drawn from PCG32's default stream).  HALTON needs spp * sample_stride < 2^32 (else PBRT_E_UNSUPPORTED). */
typedef enum PbrtSampler { PBRT_SAMPLER_SOBOL = 0, PBRT_SAMPLER_HALTON = 1 } PbrtSampler;

/* SamplerIntegrators on these kernels: Integrator "path" (src/integrators/path.rs) and Integrator "ao" (src/integrators/ao.rs:
 * ao_samples hemisphere rays from the first hit, drawn from the sampler's 2D sample array -- dimensions 5/6 of the pixel's samples
 * s * ao_samples + k). */
typedef enum PbrtIntegrator { PBRT_INTEGRATOR_PATH = 0, PBRT_INTEGRATOR_AO = 1, PBRT_INTEGRATOR_DIRECT = 2, PBRT_INTEGRATOR_WHITTED = 3 } PbrtIntegrator;
/* DirectLightingIntegrator (src/integrators/directlighting.rs:70-260) and WhittedIntegrator (src/integrators/whitted.rs:50-254):
 * emitted + direct light at every hit, then BOTH a specular-reflection and a specular-transmission ray while depth + 1 < max_depth
 * (materials are built with allow_multiple_lobes = false, so glass is SpecularReflection + SpecularTransmission).  DIRECT samples
 * every light PbrtLight.n_samples times from the sampler's 2D sample arrays ("strategy" "all", the default; directlighting.rs:52-66,
 * integrator.rs:300-355) or one light chosen uniformly ("one", integrator.rs:383-388), with MIS; WHITTED takes one sample_li per
 * light without MIS (whitted.rs:74-98). */
typedef enum PbrtDirectStrategy { PBRT_DIRECT_SAMPLE_ALL = 0, PBRT_DIRECT_SAMPLE_ONE = 1 } PbrtDirectStrategy;

/* bounds are {xmin, ymin, xmax, ymax}, max exclusive */
typedef struct PbrtRenderParams {
    int32_t sample_bounds[4];         /* Film::get_sample_bounds()            film.rs:266 */
    int32_t cropped_pixel_bounds[4];  /* Film.cropped_pixel_bounds            film.rs:176 */
    int32_t pixel_bounds[4];          /* integrator pixel_bounds: pixels outside are skipped integrator.rs:125 */
    float filter_radius[2];           /* Filter radius                        film.rs:100 */
    float filter_table[256];          /* Film.filter_table (16x16)            film.rs:201-213 */
    float max_sample_luminance;       /* +inf by default                      film.rs:96 */
    uint32_t spp;                     /* samples_per_pixel; SOBOL: AFTER the round-up to a power of two (sobol.rs:39-45) */
    uint32_t max_depth;               /* path.rs:30 */
    float rr_threshold;               /* path.rs:31 */
    uint32_t light_strategy;          /* PbrtLightStrategy */
    uint32_t flags;                   /* PBRT_RENDER_* */
    uint32_t sampler;                 /* PbrtSampler */
    uint32_t sample_at_pixel_center;  /* HALTON "samplepixelcenter" (halton.rs:245-247) */
    uint32_t integrator;              /* PbrtIntegrator */
    uint32_t ao_samples;              /* AO "nsamples" (default 64)            ao.rs:24,44 */
    uint32_t ao_cos_sample;           /* AO "cossample" (default true)         ao.rs:23 */
    uint32_t instancing;              /* PbrtInstancing */
    uint32_t direct_strategy;         /* DIRECT: PbrtDirectStrategy */
} PbrtRenderParams;

#define PBRT_RENDER_COUNT_WORK 1u    /* also fill nodes_visited / tris_tested (slower counting kernels) */
#define PBRT_RENDER_SINGLE_STREAM 2u /* one batch in flight: per-kernel times in PbrtStats are not inflated by overlap */

typedef struct PbrtStats {
    uint64_t camera_rays;    /* paths started */
    uint64_t rays;           /* BVH traversals: closest-hit + any-hit (the unit of Mrays/s) */
    uint64_t closest_rays;   /* Scene::intersect calls */
    uint64_t shadow_rays;    /* Scene::intersect_p calls */
    uint64_t nodes_visited;  /* LinearBVHNode fetches          (COUNT_WORK only) */
    uint64_t tris_tested;    /* Triangle::intersect[_p] calls  (COUNT_WORK only) */
    uint64_t light_tri_tests;/* pdf_li single-triangle tests (not counted as rays) */
    double ms_total;         /* device time of the whole render (CUDA events) */
    double ms_trace;         /* device time inside the trace kernel */
    double ms_shade;         /* device time inside the shade kernel */
    uint32_t trace_launches;
    uint32_t kernel_launches;
    /* ABI v4 */
    uint64_t shade_slots;     /* queue slots the shade kernel processed (surface hits only: a slot whose path ray missed, or whose path
                                 already ended, is finished by the sort kernel before it, pending next-event estimate included) */
    uint64_t shaded_vertices; /* of those, surface hits it shaded (PathIntegrator::li loop bodies that reached a BSDF or a null surface) */
} PbrtStats;

typedef struct PbrtScene PbrtScene;

/* Upload a flattened scene to `device` (CUDA ordinal).  Replaces the per-tile
 * scene access of integrator.rs:107-205. */
int pbrt_gpu_scene_create(const PbrtSceneDesc* desc, int device, PbrtScene** out);

/* ---- motion blur ---------------------------------------------------------------------------------------------------------------
 * A two-keyframe AnimatedTransform (src/core/transform.rs:893-940): the inputs of AnimatedTransform::new, i.e. the start and end
 * Transforms (m and m_inv of each, row-major) and TransformTimes.  The library restates AnimatedTransform::new (decompose, the
 * shortest-path flip of the end rotation) once at scene creation and AnimatedTransform::interpolate on the device. */
typedef struct PbrtAnimatedTransform {
    float start[16], start_inv[16];
    float end[16], end_inv[16];
    float start_time, end_time;
} PbrtAnimatedTransform;
/* camera: the camera's camera_to_world (api.rs:497-502), NULL = static.  Its start must equal PbrtSceneDesc.camera.camera_to_world.
 *   Each camera sample is traced at ray.time = lerp(sample.time, shutter_open, shutter_close) (perspective.rs:226) through
 *   camera_to_world interpolated at that time (AnimatedTransform::transform_ray, transform.rs:2114-2124).
 * instances: NULL, or one entry per PbrtSceneDesc.instances (api.rs:3093-3101), whose start equals PbrtInstance.m / m_inv.  An
 *   instance whose keyframes differ is PBRT_E_UNSUPPORTED in this version: animated object instances and animated shapes stay on the
 *   caller's CPU loop.
 * Keyframes or times that are not finite are PBRT_E_UNSUPPORTED; a camera keyframe whose m_inv is not the inverse of its m (up to f32
 * rounding) is PBRT_E_INVALID. */
typedef struct PbrtMotionDesc {
    const PbrtAnimatedTransform* camera;
    const PbrtAnimatedTransform* instances;
} PbrtMotionDesc;
/* pbrt_gpu_scene_create with a motion description; motion == NULL is pbrt_gpu_scene_create.  A caller detects motion blur support
 * by this symbol. */
int pbrt_gpu_scene_create_motion(const PbrtSceneDesc* desc, const PbrtMotionDesc* motion, int device, PbrtScene** out);
/* The same scene on n_devices devices in one call, for pbrt_gpu_render_multi: out[i] (an array of n_devices handles) is an ordinary
 * scene on devices[i], which every entry point accepts and pbrt_gpu_scene_destroy frees on its own, in any order.  The description
 * is validated and the host-side tables are made once; each large array (BVH nodes, triangle records, per-vertex attributes, texture
 * pyramids) crosses PCIe once in all: device i uploads its 1/n_devices slice and copies the others from their owners over peer
 * access (NVLink / NVSwitch), or from the host where a pair has none.  n_devices == 1 is pbrt_gpu_scene_create_motion; motion may
 * be NULL.  Errors: null desc / devices / out, n_devices == 0 or a device listed twice: PBRT_E_INVALID; more than 16 devices:
 * PBRT_E_UNSUPPORTED; a bad description or device: what pbrt_gpu_scene_create returns.  On any error every out[i] is NULL. */
int pbrt_gpu_scene_create_multi(const PbrtSceneDesc* desc, const PbrtMotionDesc* motion, const int* devices, uint32_t n_devices,
                                PbrtScene** out);

/* ---- camera models (ABI v4) ----------------------------------------------------------------------------------------------------
 * PbrtCamera describes a PerspectiveCamera; a PbrtCameraModel handed to pbrt_gpu_scene_create_camera selects another of rs_pbrt's
 * cameras (api.rs:1639-1689).  Every kind draws the same CameraSample (p_film, time, p_lens), traces at ray.time = lerp(sample.time,
 * shutter_open, shutter_close) and goes through camera_to_world, animated or not (PbrtMotionDesc.camera).  What each kind reads:
 *   PERSPECTIVE   PerspectiveCamera (src/cameras/perspective.rs:190-280): every field of PbrtCamera.  The model's other fields are
 *                 ignored.
 *   ORTHOGRAPHIC  OrthographicCamera (src/cameras/orthographic.rs:38-235): raster_to_camera (the caller builds it from
 *                 Transform::orthographic(0, 1), the screen window and the FULL film resolution, :47-74), camera_to_world,
 *                 lens_radius, focal_distance, the shutter.  The ray starts at raster_to_camera(p_film) along +z.  dx_camera /
 *                 dy_camera are raster_to_camera.transform_vector of the unit raster steps (:75-84).  Without a lens the
 *                 differentials are the origin shifted by dx_camera / dy_camera with the ray's direction.  With a lens both
 *                 differentials aim at ONE focus point, p_camera + dx_camera + (0,0,1) * (focal_distance / d.z) of the already
 *                 refracted d (:181-212): ry equals rx, and dy_camera is never used.
 *   ENVIRONMENT   EnvironmentCamera (src/cameras/environment.rs:92-116): camera_to_world and the shutter only.  theta = pi * p_film.y /
 *                 full_resolution[1], phi = 2 pi * p_film.x / full_resolution[0], d = (sin theta cos phi, cos theta, sin theta sin
 *                 phi) from the origin.  The ray has NO differential (differential: None), so the first hit's texture lookups are
 *                 level-0 lookups, like a later bounce's.  raster_to_camera and the lens are not read.
 * full_resolution is Film.full_resolution {x, y}: the environment camera divides by it; the crop window does not change it.
 *   REALISTIC     RealisticCamera (src/cameras/realistic.rs:198-735): only through pbrt_gpu_scene_create_lens below, which also takes
 *                 the lens system.
 * full_resolution is Film.full_resolution {x, y}: the environment and realistic cameras divide by it; the crop window does not
 * change it.  An unknown kind, and REALISTIC handed to pbrt_gpu_scene_create_camera, are PBRT_E_UNSUPPORTED; an ENVIRONMENT or
 * REALISTIC model with a zero full_resolution is PBRT_E_INVALID. */
typedef enum PbrtCameraKind {
    PBRT_CAMERA_PERSPECTIVE = 0,
    PBRT_CAMERA_ORTHOGRAPHIC = 1,
    PBRT_CAMERA_ENVIRONMENT = 2,
    PBRT_CAMERA_REALISTIC = 3
} PbrtCameraKind;
typedef struct PbrtCameraModel {
    uint32_t kind;               /* PbrtCameraKind */
    uint32_t full_resolution[2]; /* ENVIRONMENT, REALISTIC: Film.full_resolution {x, y} */
} PbrtCameraModel;
/* pbrt_gpu_scene_create_multi with a camera model; camera == NULL is the perspective camera, motion may be NULL, and n_devices == 1
 * is a single scene.  pbrt_gpu_scene_create, _create_motion and _create_multi are this call with camera == NULL.  Errors as for
 * pbrt_gpu_scene_create_multi, and those of the camera model above. */
int pbrt_gpu_scene_create_camera(const PbrtSceneDesc* desc, const PbrtMotionDesc* motion, const PbrtCameraModel* camera, const int* devices,
                                 uint32_t n_devices, PbrtScene** out);

/* ---- the realistic camera (ABI v4) ---------------------------------------------------------------------------------------------
 * RealisticCamera (src/cameras/realistic.rs) as the caller has already built it: the library computes neither the focus nor the
 * exit pupil, so it cannot disagree with the caller's CPU loop about them.  What a camera sample does (generate_ray_differential,
 * :693-735, with generate_ray :198-251):
 *   - the film point is (-x, y, 0) of Film::get_physical_extent().lerp(p_film / full_resolution) (film.rs:293-307, from diagonal);
 *   - sample_exit_pupil (:656-688): bin min(63, floor(r / (diagonal / 2) * 64)), that bin's bounds lerped by p_lens and turned by
 *     the film point's angle, on the plane z = the last element's thickness;
 *   - trace_lenses_from_film (:266-327) from the film point to that point, through Transform::scale(1, 1, -1) both ways (origin
 *     error offset included); then camera_to_world (animated or not, PbrtMotionDesc.camera) and a normalise;
 *   - weight: simple_weighting ? cos^4(theta) * area / exit_pupil_bounds[0].area() : (shutter_close - shutter_open) * (cos^4(theta) *
 *     area) / rear_z^2, cos(theta) the z of the normalised film ray, area that of the sample's bin; 0 when the ray vignettes;
 *   - the differentials shift p_film by +0.05 (-0.05 when that vignettes) in x, then in y; when neither shift of one axis passes,
 *     the whole sample's weight is 0.  So the shifted rays are always traced, textured scene or not.
 * The integrator runs li only for a weight > 0 (integrator.rs:157): a vignetted sample adds L = 0 and counts its filter weight, so
 * it darkens its pixel; PbrtStats.camera_rays counts the samples that were traced.  Every other field of the film (L * weight *
 * filter weight, integrator.rs:186) follows.  pbrt_gpu_render_samples reports li's L, unweighted.  PbrtCamera.raster_to_camera,
 * lens_radius and focal_distance are not read. */
#define PBRT_MAX_LENS_ELEMENTS 32 /* element interfaces per lens; published prescriptions have about 6-16 */
typedef struct PbrtLensElement {
    float curvature_radius; /* metres, 0 = aperture stop */
    float thickness;        /* metres; the last element's is the focused lens-film distance (focus_thick_lens, :483-499) */
    float eta;              /* 0 = air */
    float aperture_radius;  /* metres */
} PbrtLensElement;
typedef struct PbrtRealisticLens {
    const PbrtLensElement* elements;  /* RealisticCamera.element_interfaces after construction, scene side first */
    uint32_t n_elements;              /* 1 .. PBRT_MAX_LENS_ELEMENTS */
    const float* exit_pupil_bounds;   /* RealisticCamera.exit_pupil_bounds: 64 x {pmin.x, pmin.y, pmax.x, pmax.y} */
    float film_diagonal;              /* Film.diagonal, metres */
    uint32_t simple_weighting;        /* "simpleweighting" (default true) */
} PbrtRealisticLens;
/* pbrt_gpu_scene_create_camera with a realistic camera: camera->kind must be PBRT_CAMERA_REALISTIC when lens != NULL; lens == NULL
 * is pbrt_gpu_scene_create_camera.  Errors as for that call, and: a lens with another kind, n_elements == 0, a null array, a field
 * that is not finite, a zero full_resolution, a diagonal <= 0 or bounds with pmin > pmax: PBRT_E_INVALID; more than
 * PBRT_MAX_LENS_ELEMENTS elements: PBRT_E_UNSUPPORTED.  The library keeps no pointer into *lens. */
int pbrt_gpu_scene_create_lens(const PbrtSceneDesc* desc, const PbrtMotionDesc* motion, const PbrtCameraModel* camera, const PbrtRealisticLens* lens,
                               const int* devices, uint32_t n_devices, PbrtScene** out);
void pbrt_gpu_scene_destroy(PbrtScene* scene);
/* Optional (ABI v4): page-lock a host array the caller owns -- nodes, tris, a mesh's p / n / s / uv -- so that pbrt_gpu_scene_create
 * DMAs it where it lies (cudaHostRegister, portable across devices); an array that is not pinned is copied through the library's
 * own pinned staging first.  The caller unregisters before freeing the memory.  A renderer that creates the scene once per frame
 * sequence has no need for this; one that re-creates it per frame does (557 MB for the 4.3 M-triangle scene). */
int pbrt_gpu_host_register(const void* ptr, uint64_t bytes);
int pbrt_gpu_host_unregister(const void* ptr);
/* bytes copied host->device by pbrt_gpu_scene_create for this scene (bench.py's h2d_bytes_per_step); for a replica of
 * pbrt_gpu_scene_create_multi, the bytes its device received from the host (not those it copied from its peers) */
uint64_t pbrt_gpu_scene_bytes(const PbrtScene* scene);

/* Render the samples of every pixel in pixel_rect ({x0,y0,x1,y1}, a sub-rectangle
 * of sample_bounds: this rank's share) and ADD them into film_rgbw, a HOST array
 * of area(cropped_pixel_bounds)*4 floats {contrib_sum.r,g,b, filter_weight_sum}
 * per pixel (== FilmTilePixel, film.rs:57-60), row-major.  The caller then runs
 * the unchanged merge_film_tile / write_image (film.rs:346-371,437-528). */
int pbrt_gpu_render(PbrtScene* scene, const PbrtRenderParams* params, const int32_t pixel_rect[4],
                    float* film_rgbw, PbrtStats* stats);

/* Same, but the film stays in DEVICE memory (d_film_rgbw, same layout, must be
 * zero-initialised by the caller or hold a partial film to add to) and the work
 * is ordered on cuda_stream (a cudaStream_t, NULL = default stream).  Used for
 * the multi-GPU reduce (one ncclReduce(sum) of this buffer) and for
 * device-resident timing. */
int pbrt_gpu_render_device(PbrtScene* scene, const PbrtRenderParams* params, const int32_t pixel_rect[4],
                           float* d_film_rgbw, void* cuda_stream, PbrtStats* stats);

/* ---- multi-GPU (ABI v4; SURVEY.md 8e) -------------------------------------------------------------------------------------------
 * The tile space shards trivially: samples are independent (the Sobol' / Halton value depends on pixel, sample and dimension only)
 * and the scene is read-only.  The reference deals its 16x16 tiles to the worker threads in Morton order through an atomic cursor
 * (BlockQueue::new / next, src/blockqueue/mod.rs:23-36,66-73; used at src/core/integrator.rs:86-107); here tile number t of that
 * same order belongs to part t mod n_parts, so every part gets a spatially interleaved -- and therefore balanced -- share.
 *
 * pbrt_gpu_render_tiles_device: like pbrt_gpu_render_device, for part `part` of `n_parts` of the frame's tiles (one call per rank
 * when every GPU has its own process; the per-rank films are then summed by the caller, e.g. one ncclReduce). */
int pbrt_gpu_render_tiles_device(PbrtScene* scene, const PbrtRenderParams* params, uint32_t part, uint32_t n_parts, float* d_film_rgbw,
                                 void* cuda_stream, PbrtStats* stats);
/* pbrt_gpu_render_multi: the whole frame on n_scenes devices from ONE process -- what a single rs_pbrt process calls in place of
 * its Rayon tile loop.  scenes[i] is the same description created on device i (pbrt_gpu_scene_create_multi, or
 * pbrt_gpu_scene_create per device).
 * One host thread per device renders part i of n_scenes; the device of scenes[0] then sums the other films in ONE pass, reading them
 * through NVLink / NVSwitch peer access (a staged peer copy where a pair has none), and the result is ADDED into the HOST array
 * film_rgbw exactly like pbrt_gpu_render.  stats: counters summed over the devices, times = the slowest device (+ the reduce). */
int pbrt_gpu_render_multi(PbrtScene* const* scenes, uint32_t n_scenes, const PbrtRenderParams* params, float* film_rgbw, PbrtStats* stats);

/* Optional per-sample output for parity tests: radiance of every camera sample,
 * [pixel in pixel_rect row-major][sample] * 3 floats, HOST memory. */
int pbrt_gpu_render_samples(PbrtScene* scene, const PbrtRenderParams* params, const int32_t pixel_rect[4],
                            float* sample_rgb, PbrtStats* stats);

/* Scene::intersect (scene.rs:55): closest hit for n rays given as o[3n], d[3n],
 * t_max[n].  Outputs (HOST, each n long unless noted): prim = index into tris or
 * -1, t, b[3n] barycentrics. */
int pbrt_gpu_intersect(PbrtScene* scene, uint32_t n, const float* o, const float* d, const float* t_max,
                       int32_t* prim, float* t, float* b, PbrtStats* stats);

/* Scene::intersect_p (scene.rs:67): occluded[i] = 1 if anything is hit. */
int pbrt_gpu_intersect_p(PbrtScene* scene, uint32_t n, const float* o, const float* d, const float* t_max,
                         uint8_t* occluded, PbrtStats* stats);

const char* pbrt_gpu_last_error(void);
int pbrt_gpu_abi_version(void);
/* number of kernels this library has launched in this process (bench.py's gpu_launches) */
uint64_t pbrt_gpu_launch_count(void);
/* Known-answer hook: the device's f32 sin / cos (a restatement of glibc's sinf/cosf, which the reference reaches through Rust's
 * f32::sin/cos) for n arguments. Tests compare it bit for bit with the host libm. Not part of the render path. */
int pbrt_gpu_kat_sincos(int device, uint32_t n, const float* x, float* sin_out, float* cos_out);
/* Same for acos(x[i]) and atan2(y[i], x[i]) (glibc's acosf / atan2f; used by InfiniteAreaLight). */
int pbrt_gpu_kat_acos_atan2(int device, uint32_t n, const float* x, const float* y, float* acos_out, float* atan2_out);
/* Same for log2(x[i]) (glibc's log2f; MIPMap level selection). */
int pbrt_gpu_kat_log2(int device, uint32_t n, const float* x, float* log2_out);
/* Known-answer hook for motion blur: AnimatedTransform::new of *at on the host, then AnimatedTransform::interpolate on the device at
 * n times, writing 16 floats of m and 16 of m_inv per time (row-major).  Not part of the render path. */
int pbrt_gpu_kat_animated_interpolate(int device, const PbrtAnimatedTransform* at, uint32_t n, const float* times, float* m_out, float* m_inv_out);
/* Known-answer hook for the realistic camera: the device's generate_ray_differential of a scene from pbrt_gpu_scene_create_lens for n
 * camera samples (p_film[2n], p_lens[2n], time[n]), through its camera_to_world (animated or not).  Per sample: o[3], d[3], the
 * weight, and the world-space differentials rx_o / ry_o / rx_d / ry_d [3] before the 1/sqrt(spp) scale.  Where the weight is 0 the
 * rays are written as zeros.  Not part of the render path. */
int pbrt_gpu_kat_realistic_rays(PbrtScene* scene, uint32_t n, const float* p_film, const float* p_lens, const float* time, float* o, float* d,
                                float* weight, float* rx_o, float* ry_o, float* rx_d, float* ry_d);

#ifdef __cplusplus
}
#endif
#endif /* PBRT_GPU_H */
