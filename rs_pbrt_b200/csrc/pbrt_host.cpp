// pbrt_host.cpp -- C++ host mirror above the GPU C ABI (see include/pbrt_host.h for the map to the
// reference's call sequence).  Scene assembly, BVHAccel::new, PerspectiveCamera / Film set-up and the
// film merge stay on the CPU exactly as in rs_pbrt; only the per-tile loop goes to the GPU.
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <future>
#include <limits>
#include <memory>
#include <string>
#include <vector>

#include "../../include/pbrt_host.h"

namespace {

thread_local std::string g_herr;
int hfail(int code, const std::string& m) { g_herr = m; return code; }

// ---------------------------------------------------------------------------------------------
// BVHAccel::new (src/accelerators/bvh.rs:96-392), SplitMethod::SAH, built with one task per large
// subtree.  Children only touch disjoint ranges of the primitive-info array, so the tree is
// independent of the build order; the reference's observable ordering (second child's primitives
// first in `primitives`, first child first in `nodes`, quirk Q3) is applied when flattening.
struct Box3 {
    float lo[3], hi[3];
    void reset() {
        for (int k = 0; k < 3; ++k) { lo[k] = std::numeric_limits<float>::max(); hi[k] = -std::numeric_limits<float>::max(); }
    }
    void grow(const Box3& b) {
        for (int k = 0; k < 3; ++k) { lo[k] = std::fmin(lo[k], b.lo[k]); hi[k] = std::fmax(hi[k], b.hi[k]); }
    }
    void grow(const float* p) {
        for (int k = 0; k < 3; ++k) { lo[k] = std::fmin(lo[k], p[k]); hi[k] = std::fmax(hi[k], p[k]); }
    }
    float area() const {  // Bounds3f::surface_area geometry.rs:2050-2055
        float dx = hi[0] - lo[0], dy = hi[1] - lo[1], dz = hi[2] - lo[2];
        float r = dx * dy + dx * dz + dy * dz;
        return r + r;
    }
    int max_extent() const {  // geometry.rs:2056-2065
        float dx = hi[0] - lo[0], dy = hi[1] - lo[1], dz = hi[2] - lo[2];
        if (dx > dy && dx > dz) return 0;
        return dy > dz ? 1 : 2;
    }
};
struct PrimRef { uint32_t id; Box3 b; float c[3]; };
struct TreeNode { Box3 b; int32_t kid[2]; uint32_t start, end; uint8_t axis; };

struct Builder {
    std::vector<PrimRef> prims;
    std::vector<TreeNode> pool;
    std::atomic<uint32_t> next{0};
    std::atomic<int> tasks_left{0};
    uint32_t max_leaf = 4;

    static uint32_t bucket(const Box3& cb, const float* c, int dim) {
        float o = c[dim] - cb.lo[dim];  // Bounds3f::offset geometry.rs:2066-2078
        if (cb.hi[dim] > cb.lo[dim]) o /= cb.hi[dim] - cb.lo[dim];
        float v = 12.0f * o;
        int32_t bi = (v != v) ? 0 : (v >= 2147483648.0f ? 2147483647 : (v <= 0.0f ? 0 : (int32_t)v));  // `as usize`
        return bi >= 12 ? 11u : (uint32_t)bi;
    }
    uint32_t new_node() { return next.fetch_add(1); }

    uint32_t build(uint32_t start, uint32_t end) {
        const uint32_t me = new_node();
        TreeNode nd;
        nd.b.reset();
        for (uint32_t i = start; i < end; ++i) nd.b.grow(prims[i].b);
        nd.start = start; nd.end = end; nd.kid[0] = nd.kid[1] = -1; nd.axis = 0;
        const uint32_t n = end - start;
        bool leaf = n == 1;
        uint32_t mid = (start + end) / 2;
        int dim = 0;
        if (!leaf) {
            Box3 cb;
            cb.reset();
            for (uint32_t i = start; i < end; ++i) cb.grow(prims[i].c);
            dim = cb.max_extent();
            if (cb.hi[dim] == cb.lo[dim]) leaf = true;
            else if (n <= 2) {
                if (start != end - 1 && prims[end - 1].c[dim] < prims[start].c[dim]) std::swap(prims[start], prims[end - 1]);
            } else {
                uint32_t cnt[12] = {0};
                Box3 bb[12];
                for (auto& b : bb) b.reset();
                for (uint32_t i = start; i < end; ++i) {
                    uint32_t k = bucket(cb, prims[i].c, dim);
                    cnt[k]++;
                    bb[k].grow(prims[i].b);
                }
                // prefix / suffix unions: min/max are exact, so this equals the reference's O(12^2) loops
                Box3 pre[12], suf[12];
                uint32_t pc[12], sc[12];
                Box3 acc; acc.reset(); uint32_t c = 0;
                for (int k = 0; k < 12; ++k) { acc.grow(bb[k]); c += cnt[k]; pre[k] = acc; pc[k] = c; }
                acc.reset(); c = 0;
                for (int k = 11; k >= 0; --k) { acc.grow(bb[k]); c += cnt[k]; suf[k] = acc; sc[k] = c; }
                float best = 0.0f; int best_k = 0;
                const float inv_parent = nd.b.area();
                for (int k = 0; k < 11; ++k) {
                    float cost = 1.0f + ((float)pc[k] * pre[k].area() + (float)sc[k + 1] * suf[k + 1].area()) / inv_parent;
                    if (k == 0 || cost < best) { best = cost; best_k = k; }
                }
                if (n > max_leaf || best < (float)n) {
                    auto it = std::stable_partition(prims.begin() + start, prims.begin() + end,
                                                    [&](const PrimRef& r) { return bucket(cb, r.c, dim) <= (uint32_t)best_k; });
                    mid = (uint32_t)(it - prims.begin());
                } else leaf = true;
            }
        }
        if (!leaf) {
            nd.axis = (uint8_t)dim;
            pool[me] = nd;
            uint32_t k0, k1;
            if (n > 32768 && tasks_left.fetch_sub(1) > 0) {
                auto fut = std::async(std::launch::async, [this, mid, end] { return build(mid, end); });
                k0 = build(start, mid);
                k1 = fut.get();
            } else {
                k1 = build(mid, end);
                k0 = build(start, mid);
            }
            pool[me].kid[0] = (int32_t)k0;
            pool[me].kid[1] = (int32_t)k1;
            Box3 u = pool[k0].b;  // init_interior: union of the children (bvh.rs:61-67)
            u.grow(pool[k1].b);
            pool[me].b = u;
        } else pool[me] = nd;
        return me;
    }
    // assign primitive offsets in the reference's creation order: second child first
    void order_prims(uint32_t node, std::vector<uint32_t>& ordered, std::vector<uint32_t>& first) {
        std::vector<uint32_t> st{node};
        while (!st.empty()) {
            uint32_t n = st.back(); st.pop_back();
            const TreeNode& t = pool[n];
            if (t.kid[0] < 0) {
                first[n] = (uint32_t)ordered.size();
                for (uint32_t i = t.start; i < t.end; ++i) ordered.push_back(prims[i].id);
            } else { st.push_back((uint32_t)t.kid[0]); st.push_back((uint32_t)t.kid[1]); }  // kid[1] popped first
        }
    }
    uint32_t flatten(uint32_t node, const std::vector<uint32_t>& first, PbrtBvhNode* out, uint32_t& cursor) {
        const uint32_t my = cursor++;
        const TreeNode& t = pool[node];
        PbrtBvhNode ln;
        std::memset(&ln, 0, sizeof ln);
        for (int k = 0; k < 3; ++k) { ln.pmin[k] = t.b.lo[k]; ln.pmax[k] = t.b.hi[k]; }
        if (t.kid[0] < 0) {
            ln.offset = (int32_t)first[node];
            ln.n_prims = (uint16_t)(t.end - t.start);
        } else {
            flatten((uint32_t)t.kid[0], first, out, cursor);
            ln.offset = (int32_t)flatten((uint32_t)t.kid[1], first, out, cursor);
            ln.axis = t.axis;
        }
        out[my] = ln;
        return my;
    }
};

int bvh_build(const float* bounds, uint32_t n, uint32_t max_prims, int n_threads, std::vector<PbrtBvhNode>& nodes, std::vector<uint32_t>& ordered) {
    nodes.clear(); ordered.clear();
    if (n == 0) return 0;
    Builder b;
    b.max_leaf = std::min<uint32_t>(max_prims, 255);
    b.prims.resize(n);
    for (uint32_t i = 0; i < n; ++i) {
        const float* s = bounds + 6 * (size_t)i;
        PrimRef& r = b.prims[i];
        r.id = i;
        for (int k = 0; k < 3; ++k) { r.b.lo[k] = s[k]; r.b.hi[k] = s[3 + k]; r.c[k] = s[k] * 0.5f + s[3 + k] * 0.5f; }  // bvh.rs:33-40
    }
    b.pool.resize(2 * (size_t)n);
    b.tasks_left = std::max(0, n_threads - 1);
    uint32_t root = b.build(0, n);
    const uint32_t total = b.next.load();
    std::vector<uint32_t> first(total, 0);
    ordered.reserve(n);
    b.order_prims(root, ordered, first);
    nodes.resize(total);
    uint32_t cursor = 0;
    b.flatten(root, first, nodes.data(), cursor);
    return 0;
}

// ---------------------------------------------------------------------------------------------
// 4x4 matrices (src/core/transform.rs:90-256), row-major
struct M4 { float m[4][4]; };
M4 m4_identity() { M4 r; std::memset(&r, 0, sizeof r); for (int i = 0; i < 4; ++i) r.m[i][i] = 1.0f; return r; }
M4 m4_mul(const M4& a, const M4& b) {
    M4 r;
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) r.m[i][j] = a.m[i][0] * b.m[0][j] + a.m[i][1] * b.m[1][j] + a.m[i][2] * b.m[2][j] + a.m[i][3] * b.m[3][j];
    return r;
}
M4 m4_inverse(const M4& in) {  // Gauss-Jordan with full pivoting, transform.rs:128-201
    int indxc[4], indxr[4], ipiv[4] = {0, 0, 0, 0};
    M4 a = in;
    for (int i = 0; i < 4; ++i) {
        int irow = 0, icol = 0;
        float big = 0.0f;
        for (int j = 0; j < 4; ++j)
            if (ipiv[j] != 1)
                for (int k = 0; k < 4; ++k)
                    if (ipiv[k] == 0) {
                        float v = std::fabs(a.m[j][k]);
                        if (v >= big) { big = v; irow = j; icol = k; }
                    }
        ipiv[icol] += 1;
        if (irow != icol) for (int k = 0; k < 4; ++k) std::swap(a.m[irow][k], a.m[icol][k]);
        indxr[i] = irow; indxc[i] = icol;
        float pivinv = 1.0f / a.m[icol][icol];
        a.m[icol][icol] = 1.0f;
        for (int j = 0; j < 4; ++j) a.m[icol][j] *= pivinv;
        for (int j = 0; j < 4; ++j)
            if (j != icol) {
                float save = a.m[j][icol];
                a.m[j][icol] = 0.0f;
                for (int k = 0; k < 4; ++k) a.m[j][k] -= a.m[icol][k] * save;
            }
    }
    for (int j = 3; j >= 0; --j)
        if (indxr[j] != indxc[j]) for (int k = 0; k < 4; ++k) std::swap(a.m[k][indxr[j]], a.m[k][indxc[j]]);
    return a;
}
struct Xf { M4 m, inv; };
Xf xf_mul(const Xf& a, const Xf& b) { return Xf{m4_mul(a.m, b.m), m4_mul(b.inv, a.inv)}; }  // transform.rs:869-877
Xf xf_scale(float x, float y, float z) {
    Xf r{m4_identity(), m4_identity()};
    r.m.m[0][0] = x; r.m.m[1][1] = y; r.m.m[2][2] = z;
    r.inv.m[0][0] = 1.0f / x; r.inv.m[1][1] = 1.0f / y; r.inv.m[2][2] = 1.0f / z;
    return r;
}
Xf xf_translate(float x, float y, float z) {
    Xf r{m4_identity(), m4_identity()};
    r.m.m[0][3] = x; r.m.m[1][3] = y; r.m.m[2][3] = z;
    r.inv.m[0][3] = -x; r.inv.m[1][3] = -y; r.inv.m[2][3] = -z;
    return r;
}
Xf xf_perspective(float fov, float n, float f) {  // transform.rs:461-489
    M4 persp = m4_identity();
    persp.m[2][2] = f / (f - n);
    persp.m[2][3] = -f * n / (f - n);
    persp.m[3][2] = 1.0f;
    persp.m[3][3] = 0.0f;
    const float PI = 3.14159265358979323846f;
    float inv_tan_ang = 1.0f / std::tan(((PI / 180.0f) * fov) / 2.0f);
    return xf_mul(xf_scale(inv_tan_ang, inv_tan_ang, 1.0f), Xf{persp, m4_inverse(persp)});
}
void xf_point(const M4& m, const float p[3], float out[3]) {  // transform.rs:490-517
    float x = p[0], y = p[1], z = p[2];
    float xp = m.m[0][0] * x + m.m[0][1] * y + m.m[0][2] * z + m.m[0][3];
    float yp = m.m[1][0] * x + m.m[1][1] * y + m.m[1][2] * z + m.m[1][3];
    float zp = m.m[2][0] * x + m.m[2][1] * y + m.m[2][2] * z + m.m[2][3];
    float wp = m.m[3][0] * x + m.m[3][1] * y + m.m[3][2] * z + m.m[3][3];
    if (wp == 1.0f) { out[0] = xp; out[1] = yp; out[2] = zp; }
    else { float inv = 1.0f / wp; out[0] = inv * xp; out[1] = inv * yp; out[2] = inv * zp; }
}
struct D3 { float x, y, z; };
D3 d3_cross(D3 a, D3 b) {  // geometry.rs:680-692 (f64 inside)
    double ax = a.x, ay = a.y, az = a.z, bx = b.x, by = b.y, bz = b.z;
    return D3{(float)((ay * bz) - (az * by)), (float)((az * bx) - (ax * bz)), (float)((ax * by) - (ay * bx))};
}
float d3_len(D3 a) { return std::sqrt(a.x * a.x + a.y * a.y + a.z * a.z); }
D3 d3_norm(D3 a) { float inv = 1.0f / d3_len(a); return D3{a.x * inv, a.y * inv, a.z * inv}; }
void d3_coordinate_system(D3 v1, D3& v2, D3& v3) {  // geometry.rs:779-794
    if (std::fabs(v1.x) > std::fabs(v1.y)) { float inv = 1.0f / std::sqrt(v1.x * v1.x + v1.z * v1.z); v2 = D3{-v1.z * inv, 0.0f * inv, v1.x * inv}; }
    else { float inv = 1.0f / std::sqrt(v1.y * v1.y + v1.z * v1.z); v2 = D3{0.0f * inv, v1.z * inv, -v1.y * inv}; }
    v3 = d3_cross(v1, v2);
}
M4 m4_translate(float x, float y, float z) { M4 r = m4_identity(); r.m[0][3] = x; r.m[1][3] = y; r.m[2][3] = z; return r; }

struct HostMesh {
    std::vector<float> p, n, s, uv;
    std::vector<uint32_t> idx;
    uint32_t n_verts = 0;
    bool reverse_orientation = false, swaps_handedness = false;
    int material = -1;
    bool emissive = false, two_sided = false;
    uint32_t light_samples = 1;
    float L[3] = {0, 0, 0};
    int object = -1;  // >= 0: defined between ObjectBegin / ObjectEnd, only reachable through instances
    uint32_t alpha = 0, shadow_alpha = 0;  // "alpha" / "shadowalpha" float textures of the Shape (1 + texture index; api.rs:1920-1964)
};

}  // namespace

struct PbrtHost {
    std::vector<PbrtMaterial> materials;
    std::vector<PbrtTexture> textures;
    std::vector<std::vector<float>> texture_texels;
    std::vector<std::unique_ptr<HostMesh>> meshes;
    struct LightDecl { size_t before_mesh; PbrtLight l; std::shared_ptr<std::vector<float>> env; };
    struct InstanceDecl { size_t before_mesh; int object; M4 m, m_inv; bool identity; };  // ObjectInstance directives, in declaration order
    std::vector<InstanceDecl> instance_decls;
    int n_objects = 0, current_object = -1;
    std::vector<PbrtInstance> instances;  // LightSource directives, kept in declaration order with the shapes
    std::vector<LightDecl> light_decls;
    // camera / film / sampler / integrator state
    M4 camera_to_world = m4_identity();
    float transform_times[2] = {0.0f, 1.0f};  // TransformTimes (api.rs:2525-2529)
    bool have_camera_end = false;             // the camera's end keyframe (ActiveTransform EndTime at the Camera directive)
    M4 camera_to_world_end = m4_identity();
    PbrtAnimatedTransform camera_motion;      // built by pbrt_host_world_end
    PbrtMotionDesc motion;
    int xres = 1280, yres = 720;
    float crop[4] = {0, 1, 0, 1};
    std::string filter = "box";
    float filter_r[2] = {0.5f, 0.5f}, filter_alpha = 2.0f;
    float max_sample_luminance = std::numeric_limits<float>::infinity();
    bool have_camera = false;
    PbrtCamera cam;
    int pixel_samples = 16;
    uint32_t sampler = PBRT_SAMPLER_SOBOL;
    bool sample_at_pixel_center = false;
    uint32_t integrator = PBRT_INTEGRATOR_PATH, ao_samples = 64, instancing = PBRT_INSTANCING_REFERENCE;
    uint32_t direct_strategy = PBRT_DIRECT_SAMPLE_ALL, light_samples = 1;
    bool ao_cos_sample = true;
    uint32_t max_depth = 5, light_strategy = PBRT_LIGHTS_SPATIAL;
    float rr_threshold = 1.0f;
    bool have_pixel_bounds = false;
    int32_t pixel_bounds[4] = {0, 0, 0, 0};
    // built scene
    bool built = false;
    std::vector<PbrtBvhNode> nodes;
    std::vector<PbrtTri> tris;
    std::vector<PbrtMesh> mesh_descs;
    std::vector<PbrtLight> lights;
    PbrtSceneDesc desc;
    PbrtRenderParams rp;
    std::vector<float> film;  // contrib_sum rgb + filter_weight_sum, cropped bounds
};

extern "C" {

const char* pbrt_host_last_error(void) { return g_herr.c_str(); }
PbrtHost* pbrt_host_new(void) { return new PbrtHost(); }
void pbrt_host_free(PbrtHost* h) { delete h; }

int pbrt_host_add_material(PbrtHost* h, uint32_t kind, const float params[24]) {
    if (!h || !params) return hfail(PBRT_E_INVALID, "null argument");
    if (kind > PBRT_MAT_TRANSLUCENT) return hfail(PBRT_E_UNSUPPORTED, "material kind outside the GPU path");
    PbrtMaterial m;
    std::memset(&m, 0, sizeof m);
    m.kind = kind;
    std::memcpy(m.params, params, sizeof m.params);
    h->materials.push_back(m);
    return (int)h->materials.size() - 1;
}

// Material "mix" "string namedmaterial1" "string namedmaterial2" "spectrum amount" (api.rs:678-705): the two named materials exist already
int pbrt_host_add_material_mix(PbrtHost* h, int m1, int m2, const float amount[3]) {
    if (!h || !amount) return hfail(PBRT_E_INVALID, "null argument");
    const int n = (int)h->materials.size();
    if (m1 < 0 || m1 >= n || m2 < 0 || m2 >= n) return hfail(PBRT_E_INVALID, "MixMaterial names a material that does not exist (yet)");  // api.rs:683-691 panics
    PbrtMaterial m;
    std::memset(&m, 0, sizeof m);
    m.kind = PBRT_MAT_MIX;
    std::memcpy(m.params, amount, 3 * sizeof(float));
    m.params[3] = (float)m1;
    m.params[4] = (float)m2;
    h->materials.push_back(m);
    return n;
}

// spectrum.rs:1865-1871
static float inverse_gamma_convert_float(float v) {
    if (v <= 0.04045f) return v / 12.92f;
    return std::pow((v + 0.055f) * 1.0f / 1.055f, 2.4f);
}

int pbrt_host_add_texture_image(PbrtHost* h, const float* rgb, uint32_t width, uint32_t height, int float_valued, int trilinear, float max_anisotropy,
                                uint32_t wrap, float scale, int gamma, float uscale, float vscale, float udelta, float vdelta) {
    if (!h || !rgb) return hfail(PBRT_E_INVALID, "null argument");
    if (width == 0 || height == 0) return hfail(PBRT_E_INVALID, "empty image");
    if (wrap > PBRT_WRAP_CLAMP) return hfail(PBRT_E_INVALID, "unknown wrap mode");
    const int nc = float_valued ? 1 : 3;
    h->texture_texels.emplace_back((size_t)width * height * nc);
    std::vector<float>& t = h->texture_texels.back();
    for (uint32_t y = 0; y < height; ++y)  // y flip (imagemap.rs:62-70), then convert_in (:71-84) and the convert closure
        for (uint32_t x = 0; x < width; ++x) {
            float c3[3];
            for (int c = 0; c < 3; ++c) {
                float v = rgb[((size_t)(height - 1 - y) * width + x) * 3 + c];
                c3[c] = (gamma ? inverse_gamma_convert_float(v) : v) * scale;
            }
            float* o = &t[((size_t)y * width + x) * nc];
            if (float_valued) o[0] = 0.212671f * c3[0] + 0.715160f * c3[1] + 0.072169f * c3[2];  // RGBSpectrum::y, spectrum.rs:1581
            else { o[0] = c3[0]; o[1] = c3[1]; o[2] = c3[2]; }
        }
    PbrtTexture tx;
    std::memset(&tx, 0, sizeof tx);
    tx.res[0] = width; tx.res[1] = height;
    tx.texels = nullptr;  // patched in world_end (the vector of vectors may move)
    tx.channels = (uint32_t)nc;
    tx.trilinear = trilinear ? 1u : 0u;
    tx.max_anisotropy = max_anisotropy;
    tx.wrap = wrap;
    tx.su = uscale; tx.sv = vscale; tx.du = udelta; tx.dv = vdelta;
    h->textures.push_back(tx);
    return (int)h->textures.size() - 1;
}

static int add_texture_node(PbrtHost* h, uint32_t kind, uint32_t channels, const float* value, int t1, int t2, int amount) {
    PbrtTexture tx;
    std::memset(&tx, 0, sizeof tx);
    tx.kind = kind; tx.channels = channels;
    if (value) for (int c = 0; c < 3; ++c) tx.value[c] = channels == 1 ? value[0] : value[c];
    const int ops[3] = {t1, t2, amount};
    const int nc = kind == PBRT_TEX_CONSTANT ? 0 : (kind == PBRT_TEX_SCALE ? 2 : 3);
    for (int c = 0; c < nc; ++c) {
        if (ops[c] < 0 || ops[c] >= (int)h->textures.size()) return hfail(PBRT_E_INVALID, "unknown texture operand");
        if (h->textures[(size_t)ops[c]].channels != (c == 2 ? 1u : channels)) return hfail(PBRT_E_INVALID, "texture operand of the wrong type");
        tx.child[c] = (uint32_t)ops[c] + 1u;
    }
    h->textures.push_back(tx);
    h->texture_texels.emplace_back();  // keeps the two vectors aligned
    return (int)h->textures.size() - 1;
}
int pbrt_host_add_texture_constant(PbrtHost* h, const float value[3], int float_valued) {
    if (!h || !value) return hfail(PBRT_E_INVALID, "null argument");
    return add_texture_node(h, PBRT_TEX_CONSTANT, float_valued ? 1u : 3u, value, -1, -1, -1);
}
int pbrt_host_add_texture_scale(PbrtHost* h, int tex1, int tex2) {
    if (!h) return hfail(PBRT_E_INVALID, "null argument");
    if (tex1 < 0 || tex1 >= (int)h->textures.size()) return hfail(PBRT_E_INVALID, "unknown texture operand");
    return add_texture_node(h, PBRT_TEX_SCALE, h->textures[(size_t)tex1].channels, nullptr, tex1, tex2, -1);
}
int pbrt_host_add_texture_mix(PbrtHost* h, int tex1, int tex2, int amount) {
    if (!h) return hfail(PBRT_E_INVALID, "null argument");
    if (tex1 < 0 || tex1 >= (int)h->textures.size()) return hfail(PBRT_E_INVALID, "unknown texture operand");
    return add_texture_node(h, PBRT_TEX_MIX, h->textures[(size_t)tex1].channels, nullptr, tex1, tex2, amount);
}

// "mapping" "spherical" | "cylindrical" (m = world_to_texture, row-major 4x4) | "planar" (m[0..3) = v1, m[3..6) = v2, "udelta" / "vdelta" stay
// in the image call's arguments) of an image texture made by pbrt_host_add_texture_image (api.rs get_texture_mapping)
int pbrt_host_texture_mapping(PbrtHost* h, int texture, uint32_t mapping, const float* m) {
    if (!h || !m) return hfail(PBRT_E_INVALID, "null argument");
    if (texture < 0 || texture >= (int)h->textures.size() || h->textures[(size_t)texture].kind != PBRT_TEX_IMAGE) return hfail(PBRT_E_INVALID, "not an image texture");
    if (mapping < PBRT_MAP_SPHERICAL || mapping > PBRT_MAP_PLANAR) return hfail(PBRT_E_INVALID, "unknown texture mapping");
    PbrtTexture& t = h->textures[(size_t)texture];
    t.mapping = mapping;
    std::memset(t.map_m, 0, sizeof t.map_m);
    std::memcpy(t.map_m, m, (mapping == PBRT_MAP_PLANAR ? 6 : 16) * sizeof(float));
    return PBRT_OK;
}
int pbrt_host_mesh_alpha(PbrtHost* h, int mesh, int alpha_texture, int shadow_alpha_texture) {  // Shape "texture alpha" / "texture shadowalpha"
    if (!h) return hfail(PBRT_E_INVALID, "null argument");
    if (mesh < 0 || mesh >= (int)h->meshes.size()) return hfail(PBRT_E_INVALID, "unknown mesh");
    for (int t : {alpha_texture, shadow_alpha_texture}) {
        if (t < 0) continue;
        if (t >= (int)h->textures.size()) return hfail(PBRT_E_INVALID, "unknown texture");
        if (h->textures[(size_t)t].channels != 1) return hfail(PBRT_E_INVALID, "an alpha mask is a float texture");
    }
    if (h->meshes[(size_t)mesh]->emissive && (alpha_texture >= 0 || shadow_alpha_texture >= 0))
        return hfail(PBRT_E_UNSUPPORTED, "alpha mask on an emissive mesh is outside the GPU path");
    h->meshes[(size_t)mesh]->alpha = alpha_texture < 0 ? 0u : (uint32_t)alpha_texture + 1u;
    h->meshes[(size_t)mesh]->shadow_alpha = shadow_alpha_texture < 0 ? 0u : (uint32_t)shadow_alpha_texture + 1u;
    return PBRT_OK;
}
int pbrt_host_material_bump(PbrtHost* h, int material, int texture) {  // "texture bumpmap" "name"
    if (!h) return hfail(PBRT_E_INVALID, "null argument");
    if (material < 0 || material >= (int)h->materials.size()) return hfail(PBRT_E_INVALID, "unknown material");
    if (texture < 0 || texture >= (int)h->textures.size()) return hfail(PBRT_E_INVALID, "unknown texture");
    if (h->textures[(size_t)texture].channels != 1) return hfail(PBRT_E_INVALID, "a bump map is a float texture");
    h->materials[(size_t)material].bump = (uint32_t)texture + 1u;
    return PBRT_OK;
}
int pbrt_host_material_texture(PbrtHost* h, int material, int group, int texture) {
    if (!h) return hfail(PBRT_E_INVALID, "null argument");
    if (material < 0 || material >= (int)h->materials.size()) return hfail(PBRT_E_INVALID, "unknown material");
    if (texture < 0 || texture >= (int)h->textures.size()) return hfail(PBRT_E_INVALID, "unknown texture");
    PbrtMaterial& m = h->materials[(size_t)material];
    int nv = 0;
    if (pbrt_material_tex_offset(m.kind, group, &nv) < 0) return hfail(PBRT_E_UNSUPPORTED, "no such parameter group for this material kind");
    if ((uint32_t)nv != h->textures[(size_t)texture].channels) return hfail(PBRT_E_INVALID, "spectrum parameter bound to a float texture or vice versa");
    m.tex[group] = (uint32_t)texture + 1u;
    return PBRT_OK;
}

int pbrt_host_add_trianglemesh(PbrtHost* h, uint32_t n_tris, const uint32_t* indices, uint32_t n_verts, const float* P, const float* N,
                               const float* S, const float* UV, int reverse_orientation, int swaps_handedness, int material,
                               const float* emit_L, int two_sided) {
    if (!h || !indices || !P) return hfail(PBRT_E_INVALID, "null argument");
    if (material >= (int)h->materials.size()) return hfail(PBRT_E_INVALID, "unknown material");
    for (size_t i = 0; i < 3 * (size_t)n_tris; ++i)
        if (indices[i] >= n_verts) return hfail(PBRT_E_INVALID, "vertex index out of range");
    std::unique_ptr<HostMesh> m(new HostMesh());
    m->idx.assign(indices, indices + 3 * (size_t)n_tris);
    m->n_verts = n_verts;
    m->p.assign(P, P + 3 * (size_t)n_verts);
    if (N) m->n.assign(N, N + 3 * (size_t)n_verts);
    if (S) m->s.assign(S, S + 3 * (size_t)n_verts);
    if (UV) m->uv.assign(UV, UV + 2 * (size_t)n_verts);
    m->reverse_orientation = reverse_orientation != 0;
    m->swaps_handedness = swaps_handedness != 0;
    m->material = material;
    if (emit_L) { m->emissive = true; m->two_sided = two_sided != 0; m->light_samples = h->light_samples; std::memcpy(m->L, emit_L, 12); }
    if (h->current_object >= 0) {
        if (m->emissive) return hfail(PBRT_E_UNSUPPORTED, "area lights are not supported with object instancing (api.rs pbrt_shape)");
        m->object = h->current_object;
    }
    h->meshes.push_back(std::move(m));
    h->built = false;
    return (int)h->meshes.size() - 1;
}

// ObjectBegin / ObjectEnd / ObjectInstance (api.rs:3001-3109).  instance_to_world = the CTM at the ObjectInstance directive, row-major
// 4x4 (NULL = identity); its inverse is computed as Transform::new does (Gauss-Jordan, transform.rs:128-201).
int pbrt_host_object_begin(PbrtHost* h) {
    if (!h) return hfail(PBRT_E_INVALID, "null argument");
    if (h->current_object >= 0) return hfail(PBRT_E_INVALID, "ObjectBegin called inside of instance definition");
    h->current_object = h->n_objects++;
    return h->current_object;
}
int pbrt_host_instancing(PbrtHost* h, uint32_t mode) {  // PbrtInstancing: how instance hits are reported (quirk Q7)
    if (!h || mode > PBRT_INSTANCING_FIXED) return hfail(PBRT_E_INVALID, "bad instancing mode");
    h->instancing = mode;
    h->built = false;
    return 0;
}
int pbrt_host_object_end(PbrtHost* h) {
    if (!h) return hfail(PBRT_E_INVALID, "null argument");
    if (h->current_object < 0) return hfail(PBRT_E_INVALID, "ObjectEnd called outside of instance definition");
    h->current_object = -1;
    return 0;
}
int pbrt_host_object_instance(PbrtHost* h, int object, const float* instance_to_world) {
    if (!h) return hfail(PBRT_E_INVALID, "null argument");
    if (h->current_object >= 0) return hfail(PBRT_E_INVALID, "ObjectInstance can't be called inside instance definition");
    if (object < 0 || object >= h->n_objects) return hfail(PBRT_E_INVALID, "unknown object");
    PbrtHost::InstanceDecl d;
    d.before_mesh = h->meshes.size();
    d.object = object;
    d.m = m4_identity();
    if (instance_to_world) std::memcpy(d.m.m, instance_to_world, 64);
    d.m_inv = m4_inverse(d.m);
    d.identity = true;
    const M4 id = m4_identity();
    for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) if (d.m.m[i][j] != id.m[i][j]) d.identity = false;  // Transform::is_identity
    h->instance_decls.push_back(d);
    h->built = false;
    return 0;
}

int pbrt_host_look_at(PbrtHost* h, const float eye[3], const float look[3], const float up[3]) {  // transform.rs:414-451
    if (!h) return hfail(PBRT_E_INVALID, "null argument");
    M4 c2w = m4_identity();
    c2w.m[0][3] = eye[0]; c2w.m[1][3] = eye[1]; c2w.m[2][3] = eye[2]; c2w.m[3][3] = 1.0f;
    D3 dir = d3_norm(D3{look[0] - eye[0], look[1] - eye[1], look[2] - eye[2]});
    D3 upn = d3_norm(D3{up[0], up[1], up[2]});
    if (d3_len(d3_cross(upn, dir)) == 0.0f) return hfail(PBRT_E_INVALID, "up vector and viewing direction are collinear");
    D3 left = d3_norm(d3_cross(upn, dir));
    D3 new_up = d3_cross(dir, left);
    c2w.m[0][0] = left.x; c2w.m[1][0] = left.y; c2w.m[2][0] = left.z; c2w.m[3][0] = 0.0f;
    c2w.m[0][1] = new_up.x; c2w.m[1][1] = new_up.y; c2w.m[2][1] = new_up.z; c2w.m[3][1] = 0.0f;
    c2w.m[0][2] = dir.x; c2w.m[1][2] = dir.y; c2w.m[2][2] = dir.z; c2w.m[3][2] = 0.0f;
    h->camera_to_world = c2w;
    return 0;
}

int pbrt_host_transform_times(PbrtHost* h, float start, float end) {  // api.rs:2525-2529
    if (!h) return hfail(PBRT_E_INVALID, "null argument");
    h->transform_times[0] = start; h->transform_times[1] = end;
    h->built = false;
    return 0;
}

int pbrt_host_camera_motion(PbrtHost* h, const float* camera_to_world_end) {
    if (!h) return hfail(PBRT_E_INVALID, "null argument");
    h->have_camera_end = camera_to_world_end != nullptr;
    if (camera_to_world_end) std::memcpy(h->camera_to_world_end.m, camera_to_world_end, 64);
    h->built = false;
    return 0;
}

// pbrt_light_source / make_light (api.rs:769-925) for the delta lights, CTM = identity (world block)
static const float PI_F = 3.14159265358979323846f;
static void scaled_spectrum(const float v[3], const float scale[3], float out[3]) {
    for (int k = 0; k < 3; ++k) out[k] = scale ? v[k] * scale[k] : v[k] * 1.0f;
}
int pbrt_host_add_light_point(PbrtHost* h, const float from[3], const float I[3], const float scale[3]) {
    if (!h || !from || !I) return hfail(PBRT_E_INVALID, "null argument");
    PbrtLight l;
    std::memset(&l, 0, sizeof l);
    l.kind = PBRT_LIGHT_POINT;
    scaled_spectrum(I, scale, l.L);
    M4 l2w = m4_mul(m4_translate(from[0], from[1], from[2]), m4_identity());
    { const float o0[3] = {0.0f, 0.0f, 0.0f}; xf_point(l2w, o0, l.p); }  // p_light = light_to_world(0,0,0)  point.rs
    l.n_samples = h->light_samples;
    h->light_decls.push_back({h->meshes.size(), l, nullptr});
    h->built = false;
    return 0;
}
int pbrt_host_add_light_spot(PbrtHost* h, const float from[3], const float to[3], const float I[3], const float scale[3], float coneangle,
                             float conedeltaangle) {
    if (!h || !from || !to || !I) return hfail(PBRT_E_INVALID, "null argument");
    PbrtLight l;
    std::memset(&l, 0, sizeof l);
    l.kind = PBRT_LIGHT_SPOT;
    scaled_spectrum(I, scale, l.L);
    D3 dir = d3_norm(D3{to[0] - from[0], to[1] - from[1], to[2] - from[2]});
    D3 du, dv;
    d3_coordinate_system(dir, du, dv);
    M4 dz = m4_identity();
    dz.m[0][0] = du.x; dz.m[0][1] = du.y; dz.m[0][2] = du.z;
    dz.m[1][0] = dv.x; dz.m[1][1] = dv.y; dz.m[1][2] = dv.z;
    dz.m[2][0] = dir.x; dz.m[2][1] = dir.y; dz.m[2][2] = dir.z;
    M4 dz_inv = m4_inverse(dz);
    // light2world = CTM * translate(from) * inverse(dir_to_z); Transform products carry m and m_inv (transform.rs:906-916)
    M4 l2w = m4_mul(m4_mul(m4_identity(), m4_translate(from[0], from[1], from[2])), dz_inv);
    M4 w2l = m4_mul(dz, m4_mul(m4_translate(-from[0], -from[1], -from[2]), m4_identity()));
    { const float o0[3] = {0.0f, 0.0f, 0.0f}; xf_point(l2w, o0, l.p); }
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) l.w2l[3 * i + j] = w2l.m[i][j];
    const float total_width = coneangle, falloff_start = coneangle - conedeltaangle;  // spot.rs:53-54, pbrt.rs:144
    l.cos_total_width = std::cos((PI_F / 180.0f) * total_width);
    l.cos_falloff_start = std::cos((PI_F / 180.0f) * falloff_start);
    l.n_samples = h->light_samples;
    h->light_decls.push_back({h->meshes.size(), l, nullptr});
    h->built = false;
    return 0;
}
int pbrt_host_add_light_distant(PbrtHost* h, const float from[3], const float to[3], const float L[3], const float scale[3]) {
    if (!h || !from || !to || !L) return hfail(PBRT_E_INVALID, "null argument");
    PbrtLight l;
    std::memset(&l, 0, sizeof l);
    l.kind = PBRT_LIGHT_DISTANT;
    scaled_spectrum(L, scale, l.L);
    D3 w = d3_norm(D3{from[0] - to[0], from[1] - to[1], from[2] - to[2]});  // distant.rs: w_light = normalize(l2w(dir))
    l.p[0] = w.x; l.p[1] = w.y; l.p[2] = w.z;
    l.n_samples = h->light_samples;
    h->light_decls.push_back({h->meshes.size(), l, nullptr});
    h->built = false;
    return 0;
}
int pbrt_host_add_light_infinite(PbrtHost* h, const float L[3], const float scale[3], const float* texels, uint32_t width, uint32_t height,
                                 const float* light_to_world, const float* world_to_light) {
    if (!h || !L) return hfail(PBRT_E_INVALID, "null argument");
    if ((light_to_world == nullptr) != (world_to_light == nullptr)) return hfail(PBRT_E_INVALID, "light_to_world and world_to_light go together");
    PbrtLight l;
    std::memset(&l, 0, sizeof l);
    l.kind = PBRT_LIGHT_INFINITE;
    float ls[3];
    scaled_spectrum(L, scale, ls);  // make_light: L * scale (api.rs:918-948)
    std::memcpy(l.L, ls, sizeof ls);
    auto env = std::make_shared<std::vector<float>>();
    const float ident[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    if (texels) {  // texels * l, infinite.rs:113-121 / 192-199
        if (width == 0 || height == 0) return hfail(PBRT_E_INVALID, "empty environment map");
        env->resize(3 * (size_t)width * height);
        for (size_t i = 0; i < (size_t)width * height; ++i)
            for (int k = 0; k < 3; ++k) (*env)[3 * i + k] = texels[3 * i + k] * ls[k];
        l.env_res[0] = width; l.env_res[1] = height;
        std::memcpy(l.l2w, light_to_world ? light_to_world : ident, sizeof ident);
        std::memcpy(l.w2l, world_to_light ? world_to_light : ident, sizeof ident);
    } else {  // InfiniteAreaLight::default: one texel, identity transforms whatever the CTM (infinite.rs:250-300)
        env->assign(ls, ls + 3);
        l.env_res[0] = l.env_res[1] = 1;
        std::memcpy(l.l2w, ident, sizeof ident);
        std::memcpy(l.w2l, ident, sizeof ident);
    }
    l.env_texels = env->data();
    l.n_samples = h->light_samples;
    h->light_decls.push_back({h->meshes.size(), l, env});
    h->built = false;
    return 0;
}

int pbrt_host_film(PbrtHost* h, int xres, int yres, const float* crop, const char* filter_name, float xwidth, float ywidth, float filter_alpha,
                   float max_sample_luminance) {
    if (!h || xres <= 0 || yres <= 0) return hfail(PBRT_E_INVALID, "bad film resolution");
    std::string f = filter_name ? filter_name : "box";
    if (f != "box" && f != "gaussian" && f != "triangle") return hfail(PBRT_E_UNSUPPORTED, "filter outside the host mirror");
    if (!(xwidth > 0.0f) || !(ywidth > 0.0f)) return hfail(PBRT_E_INVALID, "filter width must be positive");
    h->xres = xres; h->yres = yres;
    if (crop) std::memcpy(h->crop, crop, 16);
    h->filter = f;
    h->filter_r[0] = xwidth; h->filter_r[1] = ywidth; h->filter_alpha = filter_alpha;
    h->max_sample_luminance = max_sample_luminance;
    h->built = false;
    return 0;
}

int pbrt_host_camera_perspective(PbrtHost* h, float fov, float lens_radius, float focal_distance, float shutter_open, float shutter_close,
                                 const float* screen_window) {  // perspective.rs:46-185
    if (!h) return hfail(PBRT_E_INVALID, "null argument");
    float frame = (float)h->xres / (float)h->yres;
    float sw[4];  // xmin, xmax, ymin, ymax
    if (frame > 1.0f) { sw[0] = -frame; sw[1] = frame; sw[2] = -1.0f; sw[3] = 1.0f; }
    else { sw[0] = -1.0f; sw[1] = 1.0f; sw[2] = -1.0f / frame; sw[3] = 1.0f / frame; }
    if (screen_window) std::memcpy(sw, screen_window, 16);
    Xf camera_to_screen = xf_perspective(fov, 1e-2f, 1000.0f);
    Xf scale1 = xf_scale((float)h->xres, (float)h->yres, 1.0f);
    Xf scale2 = xf_scale(1.0f / (sw[1] - sw[0]), 1.0f / (sw[2] - sw[3]), 1.0f);
    Xf translate = xf_translate(-sw[0], -sw[3], 0.0f);
    Xf screen_to_raster = xf_mul(xf_mul(scale1, scale2), translate);
    Xf raster_to_screen{screen_to_raster.inv, screen_to_raster.m};
    Xf c2s_inv{camera_to_screen.inv, camera_to_screen.m};
    Xf raster_to_camera = xf_mul(c2s_inv, raster_to_screen);
    std::memcpy(h->cam.raster_to_camera, raster_to_camera.m.m, 64);
    std::memcpy(h->cam.camera_to_world, h->camera_to_world.m, 64);
    h->cam.lens_radius = lens_radius; h->cam.focal_distance = focal_distance;
    h->cam.shutter_open = shutter_open; h->cam.shutter_close = shutter_close;
    h->have_camera = true;
    return 0;
}

int pbrt_host_sampler_sobol(PbrtHost* h, int pixel_samples) {  // sobol.rs:37-45: rounded up to a power of two
    if (!h || pixel_samples <= 0) return hfail(PBRT_E_INVALID, "bad pixel sample count");
    int v = 1;
    while (v < pixel_samples) v <<= 1;
    h->pixel_samples = v;
    h->sampler = PBRT_SAMPLER_SOBOL;
    return 0;
}
int pbrt_host_sampler_halton(PbrtHost* h, int pixel_samples, int sample_at_pixel_center) {  // halton.rs:162-172 (the crate's default sampler)
    if (!h || pixel_samples <= 0) return hfail(PBRT_E_INVALID, "bad pixel sample count");
    h->pixel_samples = pixel_samples;
    h->sampler = PBRT_SAMPLER_HALTON;
    h->sample_at_pixel_center = sample_at_pixel_center != 0;
    return 0;
}

int pbrt_host_integrator_ao(PbrtHost* h, int n_samples, int cos_sample) {  // CreateAOIntegrator api.rs:411-435 ("pixelbounds" is ignored there)
    if (!h || n_samples <= 0) return hfail(PBRT_E_INVALID, "bad integrator parameters");
    h->integrator = PBRT_INTEGRATOR_AO;
    h->ao_samples = (uint32_t)n_samples;
    h->ao_cos_sample = cos_sample != 0;
    h->have_pixel_bounds = false;
    return 0;
}
// CreateDirectLightingIntegrator (api.rs) "maxdepth" (5), "strategy" "all" | "one"; CreateWhittedIntegrator "maxdepth" (5).
// "pixelbounds" as for "path".
int pbrt_host_integrator_direct(PbrtHost* h, uint32_t max_depth, uint32_t strategy, const int32_t* pixel_bounds) {
    if (!h || strategy > PBRT_DIRECT_SAMPLE_ONE) return hfail(PBRT_E_INVALID, "bad integrator parameters");
    h->integrator = PBRT_INTEGRATOR_DIRECT;
    h->max_depth = max_depth; h->direct_strategy = strategy;
    h->have_pixel_bounds = pixel_bounds != nullptr;
    if (pixel_bounds) { h->pixel_bounds[0] = pixel_bounds[0]; h->pixel_bounds[1] = pixel_bounds[2]; h->pixel_bounds[2] = pixel_bounds[1]; h->pixel_bounds[3] = pixel_bounds[3]; }
    return 0;
}
int pbrt_host_integrator_whitted(PbrtHost* h, uint32_t max_depth, const int32_t* pixel_bounds) {
    if (!h) return hfail(PBRT_E_INVALID, "bad integrator parameters");
    h->integrator = PBRT_INTEGRATOR_WHITTED;
    h->max_depth = max_depth;
    h->have_pixel_bounds = pixel_bounds != nullptr;
    if (pixel_bounds) { h->pixel_bounds[0] = pixel_bounds[0]; h->pixel_bounds[1] = pixel_bounds[2]; h->pixel_bounds[2] = pixel_bounds[1]; h->pixel_bounds[3] = pixel_bounds[3]; }
    return 0;
}
// "nsamples" of the LightSource / AreaLightSource statements that follow (Light::get_n_samples; DirectLightingIntegrator "all")
int pbrt_host_light_samples(PbrtHost* h, uint32_t n_samples) {
    if (!h || n_samples == 0) return hfail(PBRT_E_INVALID, "bad light sample count");
    h->light_samples = n_samples;
    return 0;
}
int pbrt_host_integrator_path(PbrtHost* h, uint32_t max_depth, float rr_threshold, uint32_t light_strategy, const int32_t* pixel_bounds) {
    if (!h || light_strategy > 2) return hfail(PBRT_E_INVALID, "bad integrator parameters");
    h->integrator = PBRT_INTEGRATOR_PATH;
    h->max_depth = max_depth; h->rr_threshold = rr_threshold; h->light_strategy = light_strategy;
    h->have_pixel_bounds = pixel_bounds != nullptr;
    if (pixel_bounds) { h->pixel_bounds[0] = pixel_bounds[0]; h->pixel_bounds[1] = pixel_bounds[2]; h->pixel_bounds[2] = pixel_bounds[1]; h->pixel_bounds[3] = pixel_bounds[3]; }
    return 0;
}

int pbrt_host_world_end(PbrtHost* h, uint32_t max_prims_in_node, int n_threads) {
    if (!h) return hfail(PBRT_E_INVALID, "null argument");
    if (!h->have_camera) return hfail(PBRT_E_INVALID, "no camera");
    // ---- one GeometricPrimitive (+ DiffuseAreaLight) per triangle, one TransformedPrimitive per ObjectInstance, in declaration order
    // (api.rs:2792-2870, 3024-3109); the triangles of an object only go into that object's own BVHAccel ----
    std::vector<PbrtTri> prims;
    std::vector<PbrtLight> lights;
    std::vector<float> bounds;
    std::vector<std::vector<PbrtTri>> obj_prims((size_t)h->n_objects);
    std::vector<std::vector<float>> obj_bounds((size_t)h->n_objects);
    struct PendingInstance { size_t prim; const PbrtHost::InstanceDecl* d; };
    std::vector<PendingInstance> pending;
    h->mesh_descs.clear();
    size_t next_decl = 0, next_inst = 0;
    for (size_t mi = 0; mi <= h->meshes.size(); ++mi) {
        // render_options.lights is filled in declaration order: LightSource directives push at once (api.rs:769-925),
        // area lights when their shape is declared (api.rs:2810-2852)
        while (next_decl < h->light_decls.size() && h->light_decls[next_decl].before_mesh <= mi) lights.push_back(h->light_decls[next_decl++].l);
        while (next_inst < h->instance_decls.size() && h->instance_decls[next_inst].before_mesh <= mi) {
            PbrtTri it;
            std::memset(&it, 0, sizeof it);
            it.mesh = PBRT_MESH_INSTANCE;
            it.v[0] = (uint32_t)next_inst;
            it.material = PBRT_NO_MATERIAL;
            it.area_light = -1;
            pending.push_back({prims.size(), &h->instance_decls[next_inst]});
            prims.push_back(it);
            for (int k = 0; k < 6; ++k) bounds.push_back(0.0f);  // filled once the object's BVH root bound is known
            ++next_inst;
        }
        if (mi == h->meshes.size()) break;
        const HostMesh& m = *h->meshes[mi];
        PbrtMesh md;
        std::memset(&md, 0, sizeof md);
        md.p = m.p.data(); md.n = m.n.empty() ? nullptr : m.n.data(); md.s = m.s.empty() ? nullptr : m.s.data(); md.uv = m.uv.empty() ? nullptr : m.uv.data();
        md.n_verts = m.n_verts;
        md.reverse_orientation = m.reverse_orientation; md.transform_swaps_handedness = m.swaps_handedness;
        md.alpha = m.alpha; md.shadow_alpha = m.shadow_alpha;
        h->mesh_descs.push_back(md);
        std::vector<PbrtTri>& dst_prims = m.object >= 0 ? obj_prims[(size_t)m.object] : prims;
        std::vector<float>& dst_bounds = m.object >= 0 ? obj_bounds[(size_t)m.object] : bounds;
        for (size_t t = 0; t < m.idx.size() / 3; ++t) {
            PbrtTri tri;
            tri.v[0] = m.idx[3 * t]; tri.v[1] = m.idx[3 * t + 1]; tri.v[2] = m.idx[3 * t + 2];
            tri.mesh = (uint32_t)mi;
            tri.material = m.material < 0 ? PBRT_NO_MATERIAL : (uint32_t)m.material;
            tri.area_light = -1;
            const float* p0 = &m.p[3 * (size_t)tri.v[0]];
            const float* p1 = &m.p[3 * (size_t)tri.v[1]];
            const float* p2 = &m.p[3 * (size_t)tri.v[2]];
            if (m.emissive) {
                PbrtLight l;
                std::memset(&l, 0, sizeof l);
                l.kind = PBRT_LIGHT_DIFFUSE_AREA;
                std::memcpy(l.L, m.L, 12);
                l.two_sided = m.two_sided;
                l.n_samples = m.light_samples;
                l.tri = (uint32_t)prims.size();  // remapped to BVH order below
                D3 c = d3_cross(D3{p1[0] - p0[0], p1[1] - p0[1], p1[2] - p0[2]}, D3{p2[0] - p0[0], p2[1] - p0[1], p2[2] - p0[2]});
                l.area = 0.5f * d3_len(c);  // Triangle::area triangle.rs:667-675
                tri.area_light = (int32_t)lights.size();
                lights.push_back(l);
            }
            dst_prims.push_back(tri);
            for (int k = 0; k < 3; ++k) dst_bounds.push_back(std::fmin(std::fmin(p0[k], p1[k]), p2[k]));  // Triangle::world_bound triangle.rs:126-133
            for (int k = 0; k < 3; ++k) dst_bounds.push_back(std::fmax(std::fmax(p0[k], p1[k]), p2[k]));
        }
    }
    // ---- the objects' own BVHAccels (api.rs:3050-3080; an object with one primitive is wrapped directly there -- here it gets a
    // one-leaf tree, which only adds the leaf's slab test) ----
    std::vector<std::vector<PbrtBvhNode>> obj_nodes((size_t)h->n_objects);
    std::vector<std::vector<PbrtTri>> obj_tris((size_t)h->n_objects);
    for (int o = 0; o < h->n_objects; ++o) {
        std::vector<uint32_t> ord;
        if (obj_prims[(size_t)o].empty()) continue;
        bvh_build(obj_bounds[(size_t)o].data(), (uint32_t)obj_prims[(size_t)o].size(), max_prims_in_node, n_threads, obj_nodes[(size_t)o], ord);
        obj_tris[(size_t)o].resize(ord.size());
        for (size_t i = 0; i < ord.size(); ++i) obj_tris[(size_t)o][i] = obj_prims[(size_t)o][ord[i]];
    }
    // TransformedPrimitive::world_bound = instance_to_world.transform_bounds(object bound) (primitive.rs:212-215, transform.rs:596-652)
    for (const PendingInstance& pi : pending) {
        const std::vector<PbrtBvhNode>& on = obj_nodes[(size_t)pi.d->object];
        if (on.empty()) return hfail(PBRT_E_INVALID, "ObjectInstance of an empty object");
        const float* lo = on[0].pmin;
        const float* hi = on[0].pmax;
        const float corners[8][3] = {{lo[0], lo[1], lo[2]}, {hi[0], lo[1], lo[2]}, {lo[0], hi[1], lo[2]}, {lo[0], lo[1], hi[2]},
                                     {lo[0], hi[1], hi[2]}, {hi[0], hi[1], lo[2]}, {hi[0], lo[1], hi[2]}, {hi[0], hi[1], hi[2]}};
        float* bb = &bounds[6 * pi.prim];
        for (int c = 0; c < 8; ++c) {
            float q[3];
            xf_point(pi.d->m, corners[c], q);
            for (int k = 0; k < 3; ++k) {
                bb[k] = c == 0 ? q[k] : std::fmin(bb[k], q[k]);
                bb[3 + k] = c == 0 ? q[k] : std::fmax(bb[3 + k], q[k]);
            }
        }
    }
    std::vector<uint32_t> ordered;
    bvh_build(bounds.data(), (uint32_t)prims.size(), max_prims_in_node, n_threads, h->nodes, ordered);
    h->tris.resize(prims.size());
    std::vector<uint32_t> new_index(prims.size());
    for (size_t i = 0; i < ordered.size(); ++i) { h->tris[i] = prims[ordered[i]]; new_index[ordered[i]] = (uint32_t)i; }
    for (PbrtLight& l : lights) if (l.kind == PBRT_LIGHT_DIFFUSE_AREA) l.tri = new_index[l.tri];
    h->lights = lights;
    // append the objects' trees and triangles; child / primitive offsets become absolute
    std::vector<uint32_t> obj_root((size_t)h->n_objects, 0);
    for (int o = 0; o < h->n_objects; ++o) {
        if (obj_nodes[(size_t)o].empty()) continue;
        const uint32_t node_base = (uint32_t)h->nodes.size(), tri_base = (uint32_t)h->tris.size();
        obj_root[(size_t)o] = node_base;
        for (PbrtBvhNode n : obj_nodes[(size_t)o]) {
            n.offset += (int32_t)(n.n_prims > 0 ? tri_base : node_base);
            h->nodes.push_back(n);
        }
        h->tris.insert(h->tris.end(), obj_tris[(size_t)o].begin(), obj_tris[(size_t)o].end());
    }
    h->instances.clear();
    for (const PbrtHost::InstanceDecl& idc : h->instance_decls) {
        PbrtInstance I;
        std::memset(&I, 0, sizeof I);
        I.root = obj_root[(size_t)idc.object];
        I.identity = idc.identity ? 1u : 0u;
        std::memcpy(I.m, idc.m.m, 64);
        std::memcpy(I.m_inv, idc.m_inv.m, 64);
        h->instances.push_back(I);
    }
    PbrtSceneDesc& d = h->desc;
    std::memset(&d, 0, sizeof d);
    d.nodes = h->nodes.data(); d.n_nodes = (uint32_t)h->nodes.size();
    d.tris = h->tris.data(); d.n_tris = (uint32_t)h->tris.size();
    d.meshes = h->mesh_descs.data(); d.n_meshes = (uint32_t)h->mesh_descs.size();
    d.materials = h->materials.data(); d.n_materials = (uint32_t)h->materials.size();
    for (size_t i = 0; i < h->textures.size(); ++i) h->textures[i].texels = h->texture_texels[i].empty() ? nullptr : h->texture_texels[i].data();
    d.textures = h->textures.data(); d.n_textures = (uint32_t)h->textures.size();
    d.lights = h->lights.data(); d.n_lights = (uint32_t)h->lights.size();
    d.instances = h->instances.empty() ? nullptr : h->instances.data(); d.n_instances = (uint32_t)h->instances.size();
    d.camera = h->cam;
    // make_camera (api.rs:497-502): AnimatedTransform::new(camera_to_world.t[0], start time, camera_to_world.t[1], end time)
    std::memset(&h->motion, 0, sizeof h->motion);
    if (h->have_camera_end) {
        PbrtAnimatedTransform& a = h->camera_motion;
        M4 start;  // the camera's camera_to_world as pbrt_host_camera_perspective captured it: m and m_inv of one matrix
        std::memcpy(start.m, h->cam.camera_to_world, 64);
        const M4 inv0 = m4_inverse(start), inv1 = m4_inverse(h->camera_to_world_end);
        std::memcpy(a.start, start.m, 64); std::memcpy(a.start_inv, inv0.m, 64);
        std::memcpy(a.end, h->camera_to_world_end.m, 64); std::memcpy(a.end_inv, inv1.m, 64);
        a.start_time = h->transform_times[0]; a.end_time = h->transform_times[1];
        h->motion.camera = &a;
    }
    if (!h->nodes.empty()) for (int k = 0; k < 3; ++k) { d.world_bound[k] = h->nodes[0].pmin[k]; d.world_bound[3 + k] = h->nodes[0].pmax[k]; }  // scene.rs:28
    // ---- Film::new / get_sample_bounds (film.rs:176-223,266-289) ----
    PbrtRenderParams& rp = h->rp;
    std::memset(&rp, 0, sizeof rp);
    int32_t* cb = rp.cropped_pixel_bounds;
    cb[0] = (int32_t)std::ceil((float)h->xres * h->crop[0]); cb[2] = (int32_t)std::ceil((float)h->xres * h->crop[1]);
    cb[1] = (int32_t)std::ceil((float)h->yres * h->crop[2]); cb[3] = (int32_t)std::ceil((float)h->yres * h->crop[3]);
    rp.filter_radius[0] = h->filter_r[0]; rp.filter_radius[1] = h->filter_r[1];
    rp.sample_bounds[0] = (int32_t)std::floor((float)cb[0] + 0.5f - rp.filter_radius[0]);
    rp.sample_bounds[1] = (int32_t)std::floor((float)cb[1] + 0.5f - rp.filter_radius[1]);
    rp.sample_bounds[2] = (int32_t)std::ceil((float)cb[2] - 0.5f + rp.filter_radius[0]);
    rp.sample_bounds[3] = (int32_t)std::ceil((float)cb[3] - 0.5f + rp.filter_radius[1]);
    for (int y = 0; y < 16; ++y)
        for (int x = 0; x < 16; ++x) {
            float px = ((float)x + 0.5f) * rp.filter_radius[0] / 16.0f, py = ((float)y + 0.5f) * rp.filter_radius[1] / 16.0f;
            float v = 1.0f;  // BoxFilter::evaluate
            if (h->filter == "gaussian") {  // gaussian.rs:22-49
                float ex = std::exp(-h->filter_alpha * rp.filter_radius[0] * rp.filter_radius[0]);
                float ey = std::exp(-h->filter_alpha * rp.filter_radius[1] * rp.filter_radius[1]);
                v = std::fmax(0.0f, std::exp(-h->filter_alpha * px * px) - ex) * std::fmax(0.0f, std::exp(-h->filter_alpha * py * py) - ey);
            } else if (h->filter == "triangle")  // triangle.rs:31-34
                v = std::fmax(0.0f, rp.filter_radius[0] - std::fabs(px)) * std::fmax(0.0f, rp.filter_radius[1] - std::fabs(py));
            rp.filter_table[y * 16 + x] = v;
        }
    rp.max_sample_luminance = h->max_sample_luminance;
    rp.spp = (uint32_t)h->pixel_samples;
    rp.sampler = h->sampler;
    rp.sample_at_pixel_center = h->sample_at_pixel_center ? 1u : 0u;
    rp.integrator = h->integrator; rp.ao_samples = h->ao_samples; rp.ao_cos_sample = h->ao_cos_sample ? 1u : 0u;
    rp.direct_strategy = h->direct_strategy;
    rp.instancing = h->instancing;
    rp.max_depth = h->max_depth; rp.rr_threshold = h->rr_threshold; rp.light_strategy = h->light_strategy;
    // integrator pixel bounds: the film's sample bounds, intersected with "pixelbounds" (api.rs:287-304)
    for (int i = 0; i < 4; ++i) rp.pixel_bounds[i] = rp.sample_bounds[i];
    if (h->have_pixel_bounds) {
        rp.pixel_bounds[0] = std::max(rp.pixel_bounds[0], h->pixel_bounds[0]); rp.pixel_bounds[1] = std::max(rp.pixel_bounds[1], h->pixel_bounds[1]);
        rp.pixel_bounds[2] = std::min(rp.pixel_bounds[2], h->pixel_bounds[2]); rp.pixel_bounds[3] = std::min(rp.pixel_bounds[3], h->pixel_bounds[3]);
    }
    size_t npx = (size_t)std::max(0, cb[2] - cb[0]) * (size_t)std::max(0, cb[3] - cb[1]);
    h->film.assign(npx * 4, 0.0f);
    h->built = true;
    return 0;
}

const PbrtSceneDesc* pbrt_host_scene_desc(const PbrtHost* h) { return (h && h->built) ? &h->desc : nullptr; }
const PbrtMotionDesc* pbrt_host_motion_desc(const PbrtHost* h) { return (h && h->built && h->motion.camera) ? &h->motion : nullptr; }
const PbrtRenderParams* pbrt_host_render_params(const PbrtHost* h) { return (h && h->built) ? &h->rp : nullptr; }

int pbrt_host_render(PbrtHost* h, int device, const int32_t* pixel_rect, PbrtStats* stats) {
    if (!h || !h->built) return hfail(PBRT_E_INVALID, "pbrt_host_world_end has not run");
    PbrtScene* sc = nullptr;
    int rc = pbrt_gpu_scene_create_motion(&h->desc, pbrt_host_motion_desc(h), device, &sc);
    if (rc != PBRT_OK) return hfail(rc, pbrt_gpu_last_error());
    const int32_t* rect = pixel_rect ? pixel_rect : h->rp.sample_bounds;
    rc = pbrt_gpu_render(sc, &h->rp, rect, h->film.data(), stats);
    if (rc != PBRT_OK) g_herr = pbrt_gpu_last_error();
    pbrt_gpu_scene_destroy(sc);
    return rc;
}

const float* pbrt_host_film_rgbw(const PbrtHost* h) { return (h && h->built) ? h->film.data() : nullptr; }
int pbrt_host_film_clear(PbrtHost* h) {
    if (!h || !h->built) return hfail(PBRT_E_INVALID, "no film");
    std::fill(h->film.begin(), h->film.end(), 0.0f);
    return 0;
}
int pbrt_host_film_add_rgbw(PbrtHost* h, const float* rgbw) {
    if (!h || !h->built || !rgbw) return hfail(PBRT_E_INVALID, "no film");
    for (size_t i = 0; i < h->film.size(); ++i) h->film[i] += rgbw[i];
    return 0;
}

// merge_film_tile converts the RGB sums to XYZ (film.rs:362-367); write_image converts back and normalises (:447-470)
int pbrt_host_film_rgb(const PbrtHost* h, float* out) {
    if (!h || !h->built || !out) return hfail(PBRT_E_INVALID, "no film");
    size_t npx = h->film.size() / 4;
    for (size_t i = 0; i < npx; ++i) {
        const float* s = &h->film[4 * i];
        float xyz[3], rgb[3];
        xyz[0] = 0.412453f * s[0] + 0.357580f * s[1] + 0.180423f * s[2];  // spectrum.rs:1830-1835
        xyz[1] = 0.212671f * s[0] + 0.715160f * s[1] + 0.072169f * s[2];
        xyz[2] = 0.019334f * s[0] + 0.119193f * s[1] + 0.950227f * s[2];
        rgb[0] = 3.240479f * xyz[0] - 1.537150f * xyz[1] - 0.498535f * xyz[2];  // spectrum.rs:1823-1827
        rgb[1] = -0.969256f * xyz[0] + 1.875991f * xyz[1] + 0.041556f * xyz[2];
        rgb[2] = 0.055648f * xyz[0] - 0.204043f * xyz[1] + 1.057311f * xyz[2];
        if (s[3] != 0.0f) {
            float inv = 1.0f / s[3];
            for (int c = 0; c < 3; ++c) rgb[c] = std::fmax(rgb[c] * inv, 0.0f);
        }
        out[3 * i] = rgb[0]; out[3 * i + 1] = rgb[1]; out[3 * i + 2] = rgb[2];
    }
    return 0;
}

int pbrt_host_write_image(const PbrtHost* h, const char* path) {
    if (!h || !h->built || !path) return hfail(PBRT_E_INVALID, "no film");
    size_t npx = h->film.size() / 4;
    std::vector<float> rgb(npx * 3);
    pbrt_host_film_rgb(h, rgb.data());
    const int32_t* cb = h->rp.cropped_pixel_bounds;
    int w = cb[2] - cb[0], ht = cb[3] - cb[1];
    FILE* f = std::fopen(path, "wb");
    if (!f) return hfail(PBRT_E_INVALID, "cannot open output file");
    std::fprintf(f, "P6\n%d %d\n255\n", w, ht);
    std::vector<unsigned char> row((size_t)w * 3);
    for (int y = 0; y < ht; ++y) {
        for (int x = 0; x < 3 * w; ++x) {
            float v = rgb[(size_t)y * 3 * w + x];
            float g = (v <= 0.0031308f) ? 12.92f * v : 1.055f * std::pow(v, (float)(1.0 / 2.4)) - 0.055f;  // gamma_correct pbrt.rs:99-105
            float q = 255.0f * g + 0.5f;
            q = q < 0.0f ? 0.0f : (q > 255.0f ? 255.0f : q);
            row[x] = (unsigned char)q;
        }
        std::fwrite(row.data(), 1, row.size(), f);
    }
    std::fclose(f);
    return 0;
}

int pbrt_host_bvh_build(const float* bounds, uint32_t n, uint32_t max_prims_in_node, int n_threads, PbrtBvhNode* nodes_out,
                        uint32_t* n_nodes_out, uint32_t* ordered_out) {
    if ((n && !bounds) || !nodes_out || !n_nodes_out || !ordered_out) return hfail(PBRT_E_INVALID, "null argument");
    std::vector<PbrtBvhNode> nodes;
    std::vector<uint32_t> ordered;
    bvh_build(bounds, n, max_prims_in_node, n_threads, nodes, ordered);
    if (!nodes.empty()) std::memcpy(nodes_out, nodes.data(), nodes.size() * sizeof(PbrtBvhNode));
    if (!ordered.empty()) std::memcpy(ordered_out, ordered.data(), ordered.size() * sizeof(uint32_t));
    *n_nodes_out = (uint32_t)nodes.size();
    return 0;
}

}  // extern "C"
