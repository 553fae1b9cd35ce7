// pb_scene.cuh -- device-resident scene and wavefront state layout (see DESIGN.md "Data layout in HBM").
#pragma once
#include "pb_math.cuh"

namespace pb {

// BxDF lobe kinds (src/core/reflection.rs:462-484, in-scope subset) and type bits (:448-456)
enum LobeKind { LOBE_SPEC_REFL = 0, LOBE_SPEC_TRANS, LOBE_FRESNEL_SPEC, LOBE_LAMBERT, LOBE_OREN_NAYAR, LOBE_MF_REFL, LOBE_MF_TRANS, LOBE_FRESNEL_BLEND,
                LOBE_LAMBERT_TRANS /* LambertianTransmission (TranslucentMaterial): no specialised k_shade instantiation, always a general class */ };
enum { BSDF_REFLECTION = 1, BSDF_TRANSMISSION = 2, BSDF_DIFFUSE = 4, BSDF_GLOSSY = 8, BSDF_SPECULAR = 16, BSDF_ALL = 31 };
enum FresnelKind { FRESNEL_NOOP = 0, FRESNEL_CONDUCTOR, FRESNEL_DIELECTRIC };

struct DLobe {            // 96 bytes
    int kind, type, fresnel;
    int has_sc;           // the BxDF's sc_opt is Some(scale): only on the lobes of a MixMaterial's children (mixmat.rs:52-72).  The scale sits in
                          // the one spectrum field its lobe kind leaves unused (lobe_sc below), so that the record -- and with it every material
                          // table, k_texture's per-hit record and the specialised k_shade instantiations -- is what it was without MixMaterial
    float r[3];           // R / Kd / rd                                         | sc of a transmission-only lobe
    float t[3];           // T / rs                                              | sc of a reflection-only lobe
    float eta_a, eta_b;   // transmission lobes
    float fr_a[3];        // conductor eta_t ; dielectric {eta_i, eta_t, -}
    float fr_k[3];        // conductor k   (conductor eta_i is always 1: metal.rs:183) | sc of FresnelSpecular / FresnelBlend (r and t both taken)
    float alpha_x, alpha_y;
    float on_a, on_b;     // Oren-Nayar A, B
};
// where a lobe keeps its sc_opt: r of a lobe that only has T, t of one that only has R, fr_k of the two kinds that use both (neither has a conductor Fresnel)
PB_HD float* lobe_sc_slot(DLobe& l) {
    if (l.kind == LOBE_FRESNEL_SPEC || l.kind == LOBE_FRESNEL_BLEND) return l.fr_k;
    return (l.kind == LOBE_SPEC_TRANS || l.kind == LOBE_LAMBERT_TRANS || l.kind == LOBE_MF_TRANS) ? l.r : l.t;
}
PB_HD const float* lobe_sc_slot(const DLobe& l) { return lobe_sc_slot(const_cast<DLobe&>(l)); }
#define PB_MAX_LOBES 5
#define PB_SHADE_CLASSES 16  // class 0 = no surface to shade (miss / finished path: only the pending NEE is resolved)
struct DMaterial {
    float eta;
    int n_lobes;
    int nonspecular;      // num_components(ALL & ~SPECULAR)
    int cls;              // shading class (1..PB_SHADE_CLASSES-1): materials with the same lobe-kind sequence share one
    DLobe lobes[PB_MAX_LOBES];
};
struct DLight {           // DiffuseAreaLight over one triangle (lights/diffuse.rs:19-24) | PointLight | SpotLight | DistantLight
    float L[3];           // l_emit | I | L
    uint32_t tri;
    uint32_t two_sided;
    float area;
    uint32_t kind;        // PbrtLightKind
    float cos_total_width;
    float p[3];           // p_light | w_light
    float cos_falloff_start;
    float w2l[9];         // spot: world_to_light rotation
    uint32_t env;         // infinite: index into DScene::envs
    uint32_t n_samples;   // Light::get_n_samples (DirectLightingIntegrator "all"); the size of the struct is unchanged
    float pad;
};
// InfiniteAreaLight (lights/infinite.rs): MIP level 0 of the radiance map (every lookup the path makes has width 0 and lands on
// MipMap::triangle(0, st), mipmap.rs:233-240) and the 2w x 2h Distribution2D (sampling.rs:150-198), stored densely.
// A GonioPhotometricLight / ProjectionLight (lights/goniometric.rs, projection.rs) has the same kind of record: MIP level 0 of its
// map (w == 0: no map, scale 1) and, for a projection light, the constants of ProjectionLight::new in place of the distribution.
struct DEnv {
    const float4* texels;  // w*h, row-major, {r,g,b,_}
    int w, h;              // powers of two
    int nu, nv;            // distribution resolution (2w, 2h)
    union {
        struct {
            const float* cond_func;  // [nv][nu]
            const float* cond_cdf;   // [nv][nu+1]
            const float* cond_int;   // [nv] func_int of each row
            const float* marg_func;  // [nv]
            const float* marg_cdf;   // [nv+1]
            float marg_int;
            float l2w[9], w2l[9];
        };
        struct {
            float proj[16];     // light_projection.m, row-major (Transform::perspective(fov, hither, yon))
            float screen[4];    // screen_bounds {pmin.x, pmin.y, pmax.x, pmax.y}
            float hither;
        };
    };
};

// ImageTexture<Spectrum> (imagemap.rs:17-150): the MIP pyramid of MipMap::new, all levels in one float4 array ({r,g,b,_}, row-major,
// level l at off[l], resolution (w >> l, h >> l) clamped to >= 1), the lookup mode and the UVMapping2D.
#define PB_MAX_MIP_LEVELS 16
struct DTexture {
    const float4* texels;
    int w, h;               // level 0, powers of two
    int n_levels;
    uint32_t wrap;          // PbrtWrap
    uint32_t trilinear;
    float max_anisotropy;
    float su, sv, du, dv;
    uint32_t off[PB_MAX_MIP_LEVELS];
    uint32_t mapping;       // PbrtTextureMapping: uv | spherical | cylindrical | planar
    float map_m[16];        // world_to_texture, or planar vs / vt
    uint32_t kind;          // PbrtTextureKind: image | constant | scale | mix
    float value[3];
    uint32_t child[3];      // 1 + texture index of tex1, tex2, amount (lower than this texture's own index)
};
// A material some of whose spectrum parameters are image textures, as described (k_texture compiles it per hit)
struct DMatSrc {
    uint32_t kind;
    float params[24];
    uint32_t tex[8];        // 0 = constant, else 1 + texture index; per parameter group (pbrt_gpu.h)
    float alpha_u, alpha_v; // roughness_to_alpha done on the host (recomputed by k_texture when a roughness is textured)
    uint8_t tex_off[8];     // params[] offset of each group
    uint32_t n_spectrum;    // groups below this index are spectra, the rest floats
    uint32_t bump;          // "bumpmap": 0 = none, else 1 + float texture index
};
#define PB_MAT_BUMPED 0x200    // DMaterial.cls bit: the shading frame comes from DPaths.slot_frame[slot] as well (Material::bump ran in k_texture)
#define PB_MAT_TEXTURED 0x100  // DMaterial.cls bit: lobes come from DPaths.slot_mat[slot] (written by k_texture), not from this entry

// triangle flag bits packed in tri_verts[3*i+2].w
enum { TRI_FLIP = 1, TRI_HAS_N = 2, TRI_HAS_UV = 4, TRI_HAS_S = 8, TRI_INSTANCE = 16 /* record = {bits(instance), ...}: a TransformedPrimitive */,
       TRI_ALPHA = 32, TRI_SHADOW_ALPHA = 64 /* the mesh has an alpha_mask / shadow_alpha_mask (DScene::mesh_alpha) */ };

// One TransformedPrimitive (primitive.rs:198-272): the object's BVH root and instance_to_world / its inverse (row-major 4x4)
struct DInstance {
    uint32_t root, identity, pad0, pad1;
    float m[16], m_inv[16];
};

struct DScene {
    // BVH, 2 float4 per LinearBVHNode: {pmin.xyz, pmax.x} {pmax.yz, bits(offset), bits(n_prims | axis<<16)}
    const float4* nodes;
    uint32_t n_nodes;
    // the same tree as 64-byte records of the interior nodes with both children's boxes (k_wide_build, pb_trace.cuh::trace_rays_wide),
    // indexed like `nodes`; null when the scene does not qualify (instances, alpha masks, leaves of more than 15 primitives, ...)
    const float4* wide;
    // per triangle in BVH order, 3 float4: {p0.xyz, p1.x} {p1.yz, p2.xy} {p2.z, bits(material), bits(area_light), bits(flags)}
    const float4* tri_verts;
    uint32_t n_tris;
    // per triangle: global vertex indices (into vn/vuv/vs) {i0, i1, i2, mesh}
    const uint4* tri_idx;
    const float* vn;   // 3 per vertex (valid where the mesh has normals)
    const float* vuv;  // 2 per vertex
    const float* vs;   // 3 per vertex
    const DMaterial* materials;
    uint32_t n_materials;
    const DLight* lights;
    float world_radius;   // Bounds3f::bounding_sphere of world_bound (DistantLight::preprocess)
    uint32_t n_lights;
    const DEnv* envs;
    const DInstance* instances;
    uint32_t n_instances;
    const uint2* mesh_alpha;    // per mesh {alpha_mask, shadow_alpha_mask} as 1 + float texture index (triangle.rs:39-40); null when no mesh has one
    const DTexture* textures;   // image textures; n_textures == 0: no material is textured, k_texture is not launched
    const DMatSrc* mat_src;     // per material (meaningful where DMaterial.cls has PB_MAT_TEXTURED)
    const float* ewa_lut;       // MipMap.weight_lut (mipmap.rs:188-195), 128 entries
    uint32_t n_textures;
    float dx_camera[3], dy_camera[3];  // PerspectiveCamera::new (perspective.rs:82-99)
    uint32_t n_inf;       // scene.infinite_lights (scene.rs:36-44), as indices into lights
    uint32_t inf[4];
    float raster_to_camera[16], camera_to_world[16];
    float lens_radius, focal_distance, shutter_open, shutter_close;
    float wb_min[3], wb_max[3];
};

// Light-sampling distributions: one Distribution1D per voxel of the spatial grid
// (lightdistrib.rs:119-166), stored densely: func[v*nl + j], cdf[v*(nl+1) + j], func_int[v].
// Uniform / Power use a 1x1x1 grid whose single voxel is filled up front.
struct DLightGrid {
    int nv[3];
    int n_lights;
    int* state;        // 0 = empty, 1 = requested, 2 = ready
    float* func;
    float* cdf;
    float* func_int;
    float* contrib;    // scratch, same shape as func
    uint32_t* request; // list of requested voxels this bounce
    uint32_t* n_request;  // [0] length of the list, [1] rows handed out, [2] set when a voxel found no free row
    // When a dense nvox x n_lights table would not fit the budget (many emissive triangles), the tables hold max_rows rows that are
    // handed to voxels in the order paths first reach them -- the reference fills its voxel hash lazily in the same way
    // (lightdistrib.rs:271-377) -- and row[v] is voxel v's row.  nullptr: dense, row = v.
    int* row;
    uint32_t max_rows;
    PB_HD size_t row_of(uint32_t v) const { return row ? (size_t)row[v] : (size_t)v; }
};

// Wavefront path state, one slot per camera sample in flight.  Every field is a strided view: the sibling integrators keep one
// dense array per field (stride 1); the path integrator interleaves the fields into three 64-byte records per slot --
//   A "path"   {L + flags, ray direction, beta + eta_scale, {sampler index, dimension}}   k_raygen / k_shade write, k_sort / k_shade read
//   B "nee"    {ld_light, mis_d, mis_f, nee_beta}                                          k_shade writes, the next k_shade reads
//   C "result" {hit, mis_hit, {occl}}                                                      k_trace writes, k_sort / k_shade read
// -- because k_shade reaches the state through the class-sorted queue: slot numbers are scattered, and with twelve separate arrays
// every 16-byte field was its own 32-byte DRAM sector (far more bytes fetched per slot than used).
template <typename T> struct StridedView {
    T* p;
    uint32_t stride;  // in elements of T
    PB_HD T& operator[](size_t i) const { return p[i * stride]; }
    PB_HD explicit operator bool() const { return p != nullptr; }
};
template <typename T> inline StridedView<T> dense_view(T* p) { StridedView<T> v; v.p = p; v.stride = 1; return v; }
struct DPaths {
    StridedView<float4> ray_d;     // direction of the path ray that produced `hit` (wo = -d), -
    StridedView<float4> hit;       // written by k_trace: bits(prim) (-1 = miss), b0, b1, b2
    uint32_t* hit_inst;  // instanced scenes only: instance of that hit (0xffffffff = none); mis_inst likewise for the MIS ray
    uint32_t* mis_inst;
    StridedView<float4> beta;      // beta.rgb, eta_scale
    StridedView<float4> L;         // L.rgb, bits(flags)
    StridedView<uint2> sobol;      // 64-bit Sobol' index of this camera sample
    StridedView<uint32_t> dim;     // next Sobol' dimension
    float2* p_film;
    // next-event-estimation record written by k_shade at bounce b, resolved by k_shade at bounce b+1
    StridedView<float4> ld_light;  // f*Li*w/light_pdf of the light-sampling strategy, MIS weight of the BSDF strategy
    StridedView<uint32_t> occl;    // written by k_trace: 1 if the shadow ray is occluded
    StridedView<float4> mis_hit;   // written by k_trace: hit record of the MIS ray
    StridedView<float4> mis_d;     // MIS ray direction wi, bits(light index)
    StridedView<float4> mis_f;     // f*|wi.ns| of the BSDF-sampling strategy, scattering_pdf
    StridedView<float4> nee_beta;  // beta before the bounce, light-choice pdf
    // textured scenes only: the camera ray's (scaled) differential {rx_origin, ry_origin, rx_direction, ry_direction} as 3 float4 per slot,
    // written by k_raygen, and the lobes k_texture compiled for this slot's hit
    float4* ray_diff;
    DMaterial* slot_mat;
    float4* slot_frame;  // bump-mapped hits: {shading.n, -} {shading.dpdu, -} per slot
    float4* path_rec;    // the path integrator's interleaved record A (ray_d, beta, sobol and dim are views into it); null: dense fields
};
// bits of L.w
enum { PF_HAS_RAY = 1u, PF_HAS_SHADOW = 2u, PF_HAS_MIS = 4u, PF_SPECULAR_BOUNCE = 8u, PF_BOUNCES_SHIFT = 8 };

// Ray queue record: 2 x float4 {o.xyz, t_max} {d.xyz, bits(dest)}, dest = slot | kind << 30
enum { RAY_EXTEND = 0u, RAY_MIS = 1u, RAY_SHADOW = 2u };
#define PB_RAY_SLOT_MASK 0x3fffffffu

struct DRender {
    int sb[4], cb[4], pb[4];      // sample bounds, cropped pixel bounds, integrator pixel bounds
    int rect[4];                  // this render call's pixel rectangle
    // Tile-interleaved share of the frame (pbrt_gpu_render_tiles*): `tiles` lists this share's 16x16 tiles of sample_bounds as
    // tx | ty << 16 (integrator.rs:75-85,115-118), in the Morton order of BlockQueue::new (blockqueue/mod.rs:33-36); pixel number
    // `pix` of the share is pixel (pix & 15, (pix >> 4) & 15) of tile pix >> 8.  nullptr: the share is `rect`, row-major.
    const uint32_t* tiles;
    uint32_t n_tiles;
    uint64_t rect_w_magic;        // magic_of(rect[2] - rect[0]): share_pixel's row of a pixel number
    float filter_radius[2];
    float max_sample_luminance;
    uint32_t spp, max_depth;
    float rr_threshold;
    uint32_t log2_res, resolution;
    uint32_t light_strategy;      // effective strategy
    uint32_t instancing;          // PbrtInstancing (quirk Q7)
    // HaltonSampler (samplers/halton.rs): pixel strata and the per-dimension tables
    uint32_t halton;              // 0 = SobolSampler, 1 = HaltonSampler
    uint32_t h_center;            // sample_at_pixel_center
    uint32_t h_scale[2], h_exp[2], h_mult[2], h_stride;
    const uint4* h_dims;          // per dimension {prime, PRIME_SUMS[dim], lo, hi of ceil(2^64 / prime)}
    const uint16_t* h_perm;       // RADICAL_INVERSE_PERMUTATIONS
};

// Pixel number `pix` of this render call's share -> pixel coordinates; false for the part of an edge tile beyond sample_bounds.
PB_D bool share_pixel(const DRender& rp, uint32_t pix, int& px, int& py) {
    if (rp.tiles) {
        const uint32_t t = rp.tiles[pix >> 8];
        px = rp.sb[0] + (int)((t & 0xffffu) << 4) + (int)(pix & 15u);
        py = rp.sb[1] + (int)((t >> 16) << 4) + (int)((pix >> 4) & 15u);
        return px < rp.sb[2] && py < rp.sb[3];
    }
    const uint32_t rw = (uint32_t)(rp.rect[2] - rp.rect[0]), row = div_magic(pix, rp.rect_w_magic);
    px = rp.rect[0] + (int)(pix - row * rw);
    py = rp.rect[1] + (int)row;
    return true;
}

struct DCounters {
    unsigned long long camera_rays, closest_rays, shadow_rays, nodes_visited, tris_tested, light_tri_tests, shade_slots, shaded_vertices;
};

}  // namespace pb
