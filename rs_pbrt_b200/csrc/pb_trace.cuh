// pb_trace.cuh -- BVHAccel::intersect / intersect_p and the watertight Triangle test on the device.
//   BVHAccel::intersect      src/accelerators/bvh.rs:401-462
//   BVHAccel::intersect_p    src/accelerators/bvh.rs:463-514
//   Bounds3f::intersect_p    src/core/geometry.rs:2211-2268
//   Triangle::intersect      src/shapes/triangle.rs:134-273 (hit test part; == intersect_p :450-591)
// Traversal order (near child first by dir_is_neg[axis], 64-entry stack, leaf primitives in
// order, accept t == t_max) is kept exactly: ties between coincident hits are order dependent
// (SURVEY.md quirk Q4).
#pragma once
#include "pb_scene.cuh"

namespace pb {

struct RayPre {  // per-ray constants of the traversal and of the triangle test
    V3 o, d;
    V3 inv_dir;
    int neg[3];
    uint32_t negmask;  // bit a set when inv_dir[a] < 0
    int kx, ky, kz;
    float sx, sy, sz;
};

PB_D RayPre make_ray(V3 o, V3 d) {
    RayPre r;
    r.o = o;
    r.d = d;
    r.inv_dir = mk3(1.0f / d.x, 1.0f / d.y, 1.0f / d.z);
    r.neg[0] = r.inv_dir.x < 0.0f;
    r.neg[1] = r.inv_dir.y < 0.0f;
    r.neg[2] = r.inv_dir.z < 0.0f;
    r.negmask = (uint32_t)r.neg[0] | ((uint32_t)r.neg[1] << 1) | ((uint32_t)r.neg[2] << 2);
    r.kz = maxdim(abs3(d));
    r.kx = r.kz + 1; if (r.kx == 3) r.kx = 0;
    r.ky = r.kx + 1; if (r.ky == 3) r.ky = 0;
    float dx = comp(d, r.kx), dy = comp(d, r.ky), dz = comp(d, r.kz);
    r.sx = -dx / dz;
    r.sy = -dy / dz;
    r.sz = 1.0f / dz;
    return r;
}

PB_D bool slab_test(const float4 n0, const float4 n1, const RayPre& r, float ray_tmax) {
    const float g = 1.0f + 2.0f * gamma_n(3);
    // n0 = {pmin.x, pmin.y, pmin.z, pmax.x}, n1 = {pmax.y, pmax.z, ..}
    float t_min = ((r.neg[0] ? n0.w : n0.x) - r.o.x) * r.inv_dir.x;
    float t_max = ((r.neg[0] ? n0.x : n0.w) - r.o.x) * r.inv_dir.x;
    float ty_min = ((r.neg[1] ? n1.x : n0.y) - r.o.y) * r.inv_dir.y;
    float ty_max = ((r.neg[1] ? n0.y : n1.x) - r.o.y) * r.inv_dir.y;
    t_max *= g;
    ty_max *= g;
    if (t_min > ty_max || ty_min > t_max) return false;
    if (ty_min > t_min) t_min = ty_min;
    if (ty_max < t_max) t_max = ty_max;
    float tz_min = ((r.neg[2] ? n1.y : n0.z) - r.o.z) * r.inv_dir.z;
    float tz_max = ((r.neg[2] ? n0.z : n1.y) - r.o.z) * r.inv_dir.z;
    tz_max *= g;
    if (t_min > tz_max || tz_min > t_max) return false;
    if (tz_min > t_min) t_min = tz_min;
    if (tz_max < t_max) t_max = tz_max;
    return (t_min < ray_tmax) && (t_max > 0.0f);
}

// The same constants from their packed form {inv_dir.xyz, bits(kz | negmask << 2)} {sx, sy, sz, -} (k_rayprep computes them with
// make_ray at full lane occupancy; the persistent caster would otherwise run make_ray's six IEEE divisions for the one or two lanes
// that fetch a new ray).
PB_D void pack_ray(const RayPre& r, float4& p0, float4& p1) {
    p0 = make_float4(r.inv_dir.x, r.inv_dir.y, r.inv_dir.z, __uint_as_float((uint32_t)r.kz | (r.negmask << 2)));
    p1 = make_float4(r.sx, r.sy, r.sz, 0.0f);
}
PB_D RayPre unpack_ray(V3 o, V3 d, const float4 p0, const float4 p1) {
    RayPre r;
    r.o = o; r.d = d;
    r.inv_dir = mk3(p0.x, p0.y, p0.z);
    const uint32_t w = __float_as_uint(p0.w);
    r.kz = (int)(w & 3u);
    r.negmask = w >> 2;
    r.neg[0] = (int)(r.negmask & 1u); r.neg[1] = (int)((r.negmask >> 1) & 1u); r.neg[2] = (int)((r.negmask >> 2) & 1u);
    r.kx = r.kz + 1; if (r.kx == 3) r.kx = 0;
    r.ky = r.kx + 1; if (r.ky == 3) r.ky = 0;
    r.sx = p1.x; r.sy = p1.y; r.sz = p1.z;
    return r;
}

// The same test split in two: everything that does not depend on the ray's current t_max (`geo`, and the entry parameter t_min), so
// that slab_test(box, r, t) == slab_geo(box, r, t_min) && t_min < t for any t.  The wide traversal evaluates a far child's box when
// it visits the parent and carries t_min on its stack: comparing it with the t_max of the moment the reference would have visited
// that child reproduces the reference's decision bit for bit.
PB_D bool slab_geo(float pminx, float pminy, float pminz, float pmaxx, float pmaxy, float pmaxz, const RayPre& r, float& t_min_out) {
    const float g = 1.0f + 2.0f * gamma_n(3);
    float t_min = ((r.neg[0] ? pmaxx : pminx) - r.o.x) * r.inv_dir.x;
    float t_max = ((r.neg[0] ? pminx : pmaxx) - r.o.x) * r.inv_dir.x;
    float ty_min = ((r.neg[1] ? pmaxy : pminy) - r.o.y) * r.inv_dir.y;
    float ty_max = ((r.neg[1] ? pminy : pmaxy) - r.o.y) * r.inv_dir.y;
    t_max *= g;
    ty_max *= g;
    bool ok = !(t_min > ty_max || ty_min > t_max);
    if (ty_min > t_min) t_min = ty_min;
    if (ty_max < t_max) t_max = ty_max;
    float tz_min = ((r.neg[2] ? pmaxz : pminz) - r.o.z) * r.inv_dir.z;
    float tz_max = ((r.neg[2] ? pminz : pmaxz) - r.o.z) * r.inv_dir.z;
    tz_max *= g;
    ok = ok && !(t_min > tz_max || tz_min > t_max);
    if (tz_min > t_min) t_min = tz_min;
    if (tz_max < t_max) t_max = tz_max;
    t_min_out = t_min;
    return ok && (t_max > 0.0f);
}

struct THit { float t, b0, b1, b2; };

PB_D bool tri_test(V3 p0, V3 p1, V3 p2, const RayPre& r, float ray_tmax, THit& h) {
    V3 a = p0 - r.o, b = p1 - r.o, c = p2 - r.o;
    float p0x = comp(a, r.kx), p0y = comp(a, r.ky), p0z = comp(a, r.kz);
    float p1x = comp(b, r.kx), p1y = comp(b, r.ky), p1z = comp(b, r.kz);
    float p2x = comp(c, r.kx), p2y = comp(c, r.ky), p2z = comp(c, r.kz);
    p0x += r.sx * p0z; p0y += r.sy * p0z;
    p1x += r.sx * p1z; p1y += r.sy * p1z;
    p2x += r.sx * p2z; p2y += r.sy * p2z;
    float e0 = p1x * p2y - p1y * p2x;
    float e1 = p2x * p0y - p2y * p0x;
    float e2 = p0x * p1y - p0y * p1x;
    if (e0 == 0.0f || e1 == 0.0f || e2 == 0.0f) {  // f64 fallback at triangle edges (triangle.rs:189-200)
        double p2txp1ty = (double)p2x * (double)p1y;
        double p2typ1tx = (double)p2y * (double)p1x;
        e0 = (float)(p2typ1tx - p2txp1ty);
        double p0txp2ty = (double)p0x * (double)p2y;
        double p0typ2tx = (double)p0y * (double)p2x;
        e1 = (float)(p0typ2tx - p0txp2ty);
        double p1txp0ty = (double)p1x * (double)p0y;
        double p1typ0tx = (double)p1y * (double)p0x;
        e2 = (float)(p1typ0tx - p1txp0ty);
    }
    if ((e0 < 0.0f || e1 < 0.0f || e2 < 0.0f) && (e0 > 0.0f || e1 > 0.0f || e2 > 0.0f)) return false;
    float det = e0 + e1 + e2;
    if (det == 0.0f) return false;
    p0z *= r.sz; p1z *= r.sz; p2z *= r.sz;
    float t_scaled = e0 * p0z + e1 * p1z + e2 * p2z;
    if ((det < 0.0f && (t_scaled >= 0.0f || t_scaled < ray_tmax * det)) || (det > 0.0f && (t_scaled <= 0.0f || t_scaled > ray_tmax * det)))
        return false;
    float inv_det = 1.0f / det;
    float b0 = e0 * inv_det, b1 = e1 * inv_det, b2 = e2 * inv_det;
    float t = t_scaled * inv_det;
    // conservative t > 0 test (triangle.rs:229-273)
    float max_zt = maxcomp(abs3(mk3(p0z, p1z, p2z)));
    float delta_z = gamma_n(3) * max_zt;
    float max_xt = maxcomp(abs3(mk3(p0x, p1x, p2x)));
    float max_yt = maxcomp(abs3(mk3(p0y, p1y, p2y)));
    float delta_x = gamma_n(5) * (max_xt + max_zt);
    float delta_y = gamma_n(5) * (max_yt + max_zt);
    float delta_e = 2.0f * (gamma_n(2) * max_xt * max_yt + delta_y * max_xt + delta_x * max_yt);
    float max_e = maxcomp(abs3(mk3(e0, e1, e2)));
    float delta_t = 3.0f * (gamma_n(3) * max_e * max_zt + delta_e * max_zt + delta_z * max_e) * fabsf(inv_det);
    if (t <= delta_t) return false;
    h.t = t; h.b0 = b0; h.b1 = b1; h.b2 = b2;
    return true;
}

PB_D void load_tri(const float4* __restrict__ tv, uint32_t i, V3& p0, V3& p1, V3& p2) {
    float4 a = __ldg(tv + 3 * (size_t)i), b = __ldg(tv + 3 * (size_t)i + 1), c = __ldg(tv + 3 * (size_t)i + 2);
    p0 = mk3(a.x, a.y, a.z);
    p1 = mk3(a.w, b.x, b.y);
    p2 = mk3(b.z, b.w, c.x);
}

struct WorkCount { uint32_t nodes, tris; };

#ifndef PB_SMEM_STACK_ENTRIES
#define PB_SMEM_STACK_ENTRIES 24  // stack entries per thread kept in shared memory by the global-memory variant
#endif
#define PB_TRACE_THREADS_ 128  // == PB_TRACE_THREADS (pb_kernels.cuh)
#ifndef PB_LEAF_MIN
#define PB_LEAF_MIN 1  // lanes that must hold a leaf before the warp runs the triangle phase
#endif
#ifndef PB_FLAT_WALK
#define PB_FLAT_WALK 1  // branch-free node visit (see trace_rays); 0 = the three-branch form, kept for A/B runs
#endif
#ifndef PB_REFILL_MIN
#define PB_REFILL_MIN 1  // idle lanes a warp collects before it fetches new rays (the fetch + make_ray run at the idle lanes' occupancy)
#endif
#ifndef PB_WALK_STEPS
#define PB_WALK_STEPS 16  // node visits per lane and round before the warp re-synchronises
#endif

// 128-bit read-only global loads with L1 eviction hints: BVH nodes are re-visited by many rays (keep), leaf
// triangles and ray records are streamed (do not displace nodes).
#ifndef PB_CACHE_HINTS
#define PB_CACHE_HINTS 1
#endif
PB_D float4 ldg4_keep(const float4* p) {
#if PB_CACHE_HINTS
    float4 v;
    asm volatile("ld.global.nc.L1::evict_last.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
    return v;
#else
    return __ldg(p);
#endif
}
PB_D float4 ldg4_stream(const float4* p) {
#if PB_CACHE_HINTS
    float4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
    return v;
#else
    return __ldg(p);
#endif
}
PB_D float4 lds4(const float4* p) {  // explicit 128-bit shared-memory load
#ifdef PB_HOST_EMU
    return *p;
#else
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"((uint32_t)__cvta_generic_to_shared(p)));
    return v;
#endif
}

// -----------------------------------------------------------------------------------------------
// Persistent ray caster: every lane owns ONE ray at a time.
//
// The reference's loop (bvh.rs:421-460) is kept per ray -- same node visit order, same leaf
// primitive order, same running t_max -- but the warp executes it "while-while": all lanes first
// walk interior nodes until each has reached a leaf that passes the slab test (or has finished),
// then all lanes with a leaf run the (expensive) watertight triangle tests together.  A lane whose
// ray finishes takes the next ray from the queue (warp-aggregated atomic) instead of idling, so
// warps stay full until the queue is empty.  None of this changes which nodes a ray visits or in
// which order hits are accepted, so results and work counters equal the reference's.
//
// MODE 0: wavefront queue records {o,t_max}{d,dest}; results go to ps.hit / ps.mis_hit / ps.occl
// MODE 1: API closest hit (flat o/d/tmax arrays -> prim,t,b)      MODE 2: API any hit (-> occluded)
// Transform::transform_ray (transform.rs:538-594, point with error :662-708) by a row-major 4x4: the object-space ray of an instance
PB_D void xf_ray_dev(const float* __restrict__ m, V3 o, V3 d, float& t_max, V3& o_out, V3& d_out) {
    const float x = o.x, y = o.y, z = o.z;
    V3 ow = mk3(m[0] * x + m[1] * y + m[2] * z + m[3], m[4] * x + m[5] * y + m[6] * z + m[7], m[8] * x + m[9] * y + m[10] * z + m[11]);
    const float wp = m[12] * x + m[13] * y + m[14] * z + m[15];
    const V3 o_err = mk3(fabsf(m[0] * x) + fabsf(m[1] * y) + fabsf(m[2] * z) + fabsf(m[3]), fabsf(m[4] * x) + fabsf(m[5] * y) + fabsf(m[6] * z) + fabsf(m[7]),
                         fabsf(m[8] * x) + fabsf(m[9] * y) + fabsf(m[10] * z) + fabsf(m[11])) * gamma_n(3);
    if (wp != 1.0f) { const float inv = 1.0f / wp; ow = mk3(inv * ow.x, inv * ow.y, inv * ow.z); }
    const V3 dw = mk3(m[0] * d.x + m[1] * d.y + m[2] * d.z, m[4] * d.x + m[5] * d.y + m[6] * d.z, m[8] * d.x + m[9] * d.y + m[10] * d.z);
    const float ls = len2(dw);
    if (ls > 0.0f) {
        const float dt = dot3(abs3(dw), o_err) / ls;
        ow = ow + dw * dt;
        t_max -= dt;
    }
    o_out = ow;
    d_out = dw;
}

struct TraceIO {
    const uint32_t* perm;    // MODE 0: optional coherence order of the ray queue (k_ray_scatter), else nullptr
    uint32_t* hit_inst;      // INST: instance of the reported hit (0xffffffff = none), indexed like hit / mis_hit
    uint32_t* mis_inst;
    uint32_t instancing;     // PbrtInstancing
    const float4* rays;      // MODE 0: 2 per ray
    const float4* pre;       // MODE 0, optional: per-ray traversal constants written by k_rayprep (2 per ray), else nullptr
    const float* o;          // MODE 1/2
    const float* d;
    const float* tmax;
    StridedView<float4> hit;     // MODE 0 outputs (indexed by slot; views of DPaths)
    StridedView<float4> mis_hit;
    StridedView<uint32_t> occl;
    int* out_prim;           // MODE 1 outputs (indexed by ray)
    float* out_t;
    float* out_b;
    unsigned char* out_occ;  // MODE 2
};

// INST: the scene holds TransformedPrimitives (primitive.rs:198-272).  A leaf record with TRI_INSTANCE sends the lane into the
// object's tree with the ray of Transform::inverse(instance_to_world).transform_ray(r); the resume point of the interrupted leaf and
// a sentinel go on the same stack, and popping the sentinel brings the world ray back.  What is reported follows
// TransformedPrimitive::intersect in the selected PbrtInstancing mode (quirk Q7): `best` is the interaction as the reference last
// wrote it, `hit_flag` the value BVHAccel::intersect returns.
#define PB_SENTINEL 0xffffffffu
// ALPHA: some mesh has an alpha / shadow-alpha mask.  An accepted candidate of such a mesh is then put to the texture test of
// Triangle::intersect (alpha_mask, triangle.rs:313-330) or Triangle::intersect_p (both masks, triangle.rs:593-654); defined in
// pb_kernels.cuh, where the texture code is visible.
__device__ bool alpha_rejects(const DScene& sc, uint32_t prim, V3 p0, V3 p1, V3 p2, float b0, float b1, float b2, uint32_t flags, bool any_hit);
template <bool COUNT, int MODE, bool SMEM, bool INST = false, bool ALPHA = false>
PB_D void trace_rays(const DScene& sc, const float4* __restrict__ nodes, const float4* __restrict__ tris, const TraceIO& io, uint32_t n_rays,
                     uint32_t* __restrict__ cursor, DCounters* cnt) {
    const unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    const float inf = __int_as_float(0x7f800000);
    // Traversal stack (64 entries, bvh.rs:420).  When nodes come from global memory the hot top of the stack lives in
    // shared memory (one column per thread: conflict free) and only deeper entries spill to local memory: local
    // memory is cached in L1, where 32 warps x ~20 live entries x 128 B displaced the very BVH nodes the traversal
    // wants to find there (4.3 M-triangle scene: k_trace -26 %).  When the whole scene is shared-memory resident
    // (SMEM) there is nothing to protect in L1 and the plain local stack is faster.
    constexpr int NS = SMEM ? 0 : PB_SMEM_STACK_ENTRIES;
    __shared__ uint32_t s_stack[NS > 0 ? NS : 1][PB_TRACE_THREADS_];
    uint32_t stack[(INST ? 136 : 64) - NS];  // INST: the world tree's 64 + the object's 64 + 3 resume entries (+ padding)
    // INST: the world ray's traversal constants wait in shared memory while the lane is inside an instance, so that leaving it is
    // thirteen loads rather than re-reading the ray record and re-deriving them (make_ray: six IEEE divisions)
    __shared__ float s_world[INST ? 13 : 1][PB_TRACE_THREADS_];
#define PB_SAVE_WORLD()                                                                                                      \
    do {                                                                                                                     \
        if (INST) {                                                                                                          \
            const int t_ = threadIdx.x;                                                                                      \
            s_world[0][t_] = r.o.x; s_world[1][t_] = r.o.y; s_world[2][t_] = r.o.z;                                          \
            s_world[INST ? 3 : 0][t_] = r.d.x; s_world[INST ? 4 : 0][t_] = r.d.y; s_world[INST ? 5 : 0][t_] = r.d.z;          \
            s_world[INST ? 6 : 0][t_] = r.inv_dir.x; s_world[INST ? 7 : 0][t_] = r.inv_dir.y; s_world[INST ? 8 : 0][t_] = r.inv_dir.z; \
            s_world[INST ? 9 : 0][t_] = r.sx; s_world[INST ? 10 : 0][t_] = r.sy; s_world[INST ? 11 : 0][t_] = r.sz;            \
            s_world[INST ? 12 : 0][t_] = __uint_as_float((uint32_t)r.kz | (r.negmask << 2));                                 \
        }                                                                                                                    \
    } while (0)
#define PB_RESTORE_WORLD()                                                                                                   \
    do {                                                                                                                     \
        const int t_ = threadIdx.x;                                                                                          \
        r = unpack_ray(mk3(s_world[0][t_], s_world[INST ? 1 : 0][t_], s_world[INST ? 2 : 0][t_]),                             \
                       mk3(s_world[INST ? 3 : 0][t_], s_world[INST ? 4 : 0][t_], s_world[INST ? 5 : 0][t_]),                  \
                       make_float4(s_world[INST ? 6 : 0][t_], s_world[INST ? 7 : 0][t_], s_world[INST ? 8 : 0][t_], s_world[INST ? 12 : 0][t_]), \
                       make_float4(s_world[INST ? 9 : 0][t_], s_world[INST ? 10 : 0][t_], s_world[INST ? 11 : 0][t_], 0.0f));  \
    } while (0)
#define PB_PUSH(v) do { if (NS > 0 && sp < (uint32_t)NS) s_stack[sp][threadIdx.x] = (v); else stack[sp - NS] = (v); ++sp; } while (0)
#define PB_POP() (--sp, (NS > 0 && sp < (uint32_t)NS) ? s_stack[sp][threadIdx.x] : stack[sp - NS])
// next node to visit; in INST mode popping the sentinel leaves the instance (TransformedPrimitive::intersect's epilogue) and resumes
// the interrupted world leaf
#define PB_NEXT()                                                                                                            \
    do {                                                                                                                     \
        for (;;) {                                                                                                           \
            if (sp == 0) { done = true; break; }                                                                             \
            const uint32_t v_ = PB_POP();                                                                                    \
            if (!INST || v_ != PB_SENTINEL) { cur = v_; break; }                                                             \
            leaf_n = PB_POP();                                                                                               \
            leaf_off = PB_POP();                                                                                             \
            if (inst_hit) {                                                                                                  \
                t_max_w = t_max; /* r.t_max.set(ray.t_max.get()): the OBJECT ray's parameter, as written */                  \
                if (io.instancing == 1u || !sc.instances[cur_inst].identity) hit_flag = true;                                \
            }                                                                                                                \
            PB_RESTORE_WORLD();                                                                                              \
            t_max = t_max_w;                                                                                                 \
            cur_inst = -1;                                                                                                   \
            if (leaf_n) break; /* more primitives of the interrupted leaf */                                                 \
        }                                                                                                                    \
    } while (0)
    RayPre r;
    float t_max = 0.0f;
    THit best;
    int best_prim = -1;
    uint32_t sp = 0, cur = 0, dest = 0, leaf_off = 0, leaf_n = 0, ray_id = 0;
    bool active = false, any_hit = false, exhausted = n_rays == 0;
    // INST state: the instance being traversed, whether it produced a candidate, the world ray's t_max while inside, the ray's source
    int cur_inst = -1, best_inst = -1;
    bool inst_hit = false, hit_flag = false;
    float t_max_w = 0.0f;
    uint32_t ray_src = 0;
    uint32_t n_closest = 0, n_shadow = 0;
    WorkCount wc;
    wc.nodes = 0; wc.tris = 0;
    for (;;) {
        // ---- refill idle lanes ------------------------------------------------------------------
        unsigned idle = __ballot_sync(FULL, !active);
        if (idle && !exhausted && (PB_REFILL_MIN <= 1 || (uint32_t)__popc(idle) >= PB_REFILL_MIN || idle == FULL)) {
            uint32_t base = 0;
            if (lane == 0) base = atomicAdd(cursor, (uint32_t)__popc(idle));
            base = __shfl_sync(FULL, base, 0);
            if (base >= n_rays) exhausted = true;
            uint32_t my = base + (uint32_t)__popc(idle & ((1u << lane) - 1u));
            if (!active && my < n_rays) {
                V3 o, d;
                if (MODE == 0) {
                    const uint32_t qi = io.perm ? __ldg(io.perm + my) : my;
                    ray_src = qi;
                    float4 a = ldg4_stream(io.rays + 2 * (size_t)qi), b = ldg4_stream(io.rays + 2 * (size_t)qi + 1);
                    o = mk3(a.x, a.y, a.z); d = mk3(b.x, b.y, b.z);
                    t_max = a.w;
                    dest = __float_as_uint(b.w);
                    any_hit = (dest >> 30) == RAY_SHADOW;
                } else {
                    o = mk3(io.o[3 * (size_t)my], io.o[3 * (size_t)my + 1], io.o[3 * (size_t)my + 2]);
                    d = mk3(io.d[3 * (size_t)my], io.d[3 * (size_t)my + 1], io.d[3 * (size_t)my + 2]);
                    t_max = io.tmax[my];
                    any_hit = MODE == 2;
                    ray_src = my;
                }
                cur_inst = -1; best_inst = -1; inst_hit = false; hit_flag = false;
                ray_id = my;
                if (MODE == 0 && io.pre) r = unpack_ray(o, d, ldg4_stream(io.pre + 2 * (size_t)ray_src), ldg4_stream(io.pre + 2 * (size_t)ray_src + 1));
                else r = make_ray(o, d);
                best_prim = -1;
                best.t = 0.0f; best.b0 = best.b1 = best.b2 = 0.0f;
                sp = 0; cur = 0; leaf_n = 0;
                active = true;
                if (any_hit) n_shadow++; else n_closest++;
                if (sc.n_nodes == 0) leaf_n = 0xffffffffu;  // empty aggregate: finish immediately (bvh.rs:402-404)
            }
        }
        if (!__any_sync(FULL, active)) break;
        bool done = active && leaf_n == 0xffffffffu;
        if (done) leaf_n = 0;
        // ---- node phase: each lane walks towards its next accepted leaf, for at most PB_WALK_STEPS node visits
        // per round, so that lanes which reached a leaf or finished their ray are served (triangle tests /
        // new ray) without waiting for the longest walk in the warp; unfinished walks continue next round.
        for (int step = 0; step < PB_WALK_STEPS; ++step) {
            const bool walking = active && !done && leaf_n == 0;
            if (!walking) break;
            {
                float4 n0, n1;
                if (SMEM) { n0 = lds4(nodes + 2 * cur); n1 = lds4(nodes + 2 * cur + 1); }
                else { n0 = ldg4_keep(nodes + 2 * (size_t)cur); n1 = ldg4_keep(nodes + 2 * (size_t)cur + 1); }
                if (COUNT) wc.nodes++;
                if (PB_FLAT_WALK) {
                    // One instruction stream for the three outcomes of a visit (box missed -> pop, interior -> push far child and
                    // descend, leaf -> hand over to the leaf phase): as separate branches they ran one after the other at 6-10
                    // active lanes and took a large share of the kernel's issue slots on the 4.3 M-triangle scene; here
                    // they are selects around one predicated stack store and one stack load.
                    const bool hit = slab_test(n0, n1, r, t_max);
                    const uint32_t meta = __float_as_uint(n1.w), offset = __float_as_uint(n1.z);
                    const uint32_t n_prims = meta & 0xffffu;
                    const bool neg = ((r.negmask >> ((meta >> 16) & 3u)) & 1u) != 0u;
                    const uint32_t c_near = neg ? offset : cur + 1u, c_far = neg ? cur + 1u : offset;
                    const bool interior = hit && n_prims == 0u;
                    uint32_t top = 0u;  // the entry a miss pops
                    if (!hit && sp > 0u) top = (NS > 0 && sp - 1u < (uint32_t)NS) ? s_stack[NS > 0 ? sp - 1u : 0u][threadIdx.x] : stack[sp - 1u - NS];
                    if (interior) { if (NS > 0 && sp < (uint32_t)NS) s_stack[NS > 0 ? sp : 0u][threadIdx.x] = c_far; else stack[sp - NS] = c_far; }
                    done = !hit && sp == 0u;
                    leaf_off = hit ? offset : leaf_off;
                    leaf_n = hit ? n_prims : 0u;
                    cur = interior ? c_near : (hit ? cur : top);
                    sp = sp + (interior ? 1u : 0u) - ((!hit && sp > 0u) ? 1u : 0u);
                    if (INST && !hit && top == PB_SENTINEL) {
                        // the popped entry was the sentinel: the object's tree is exhausted.  TransformedPrimitive::intersect's epilogue,
                        // then the rest of the interrupted world leaf, or the next world node
                        leaf_n = PB_POP();
                        leaf_off = PB_POP();
                        if (inst_hit) {
                            t_max_w = t_max;  // r.t_max.set(ray.t_max.get()): the OBJECT ray's parameter, as written
                            if (io.instancing == 1u || !sc.instances[cur_inst].identity) hit_flag = true;
                        }
                        PB_RESTORE_WORLD();
                        t_max = t_max_w;
                        cur_inst = -1;
                        if (leaf_n == 0u) {
                            if (sp == 0u) done = true;
                            else cur = PB_POP();
                        }
                    }
                } else {
                    bool pop = true;
                    if (slab_test(n0, n1, r, t_max)) {
                        uint32_t meta = __float_as_uint(n1.w);
                        uint32_t offset = __float_as_uint(n1.z);
                        pop = false;
                        if (meta & 0xffffu) {
                            leaf_off = offset;
                            leaf_n = meta & 0xffffu;
                        } else {
                            uint32_t far_child;
                            if ((r.negmask >> ((meta >> 16) & 3u)) & 1u) { far_child = cur + 1; cur = offset; }
                            else { far_child = offset; cur = cur + 1; }
                            PB_PUSH(far_child);
                        }
                    }
                    if (pop) PB_NEXT();
                }
            }
        }
        // ---- leaf phase: triangle tests of the accepted leaf, in primitive order.  The tests are ~4x the cost
        // of a node visit, so they are postponed until at least PB_LEAF_MIN lanes hold a leaf -- unless nobody in
        // the warp can make progress otherwise (no walker left and nothing to refill).
        const unsigned leafm = __ballot_sync(FULL, active && leaf_n != 0);
        const unsigned walkm = __ballot_sync(FULL, active && !done && leaf_n == 0);
        const unsigned freem = __ballot_sync(FULL, !active || done);
        const bool run_leaves = (uint32_t)__popc(leafm) >= PB_LEAF_MIN || (walkm == 0u && (freem == 0u || exhausted));
        bool entered = false;
        if (run_leaves && active && leaf_n) {
            for (uint32_t i = 0; i < leaf_n; ++i) {
                V3 p0, p1, p2;
                float4 c;
                if (SMEM) {
                    float4 a = lds4(tris + 3 * (leaf_off + i)), b = lds4(tris + 3 * (leaf_off + i) + 1);
                    c = lds4(tris + 3 * (leaf_off + i) + 2);
                    p0 = mk3(a.x, a.y, a.z); p1 = mk3(a.w, b.x, b.y); p2 = mk3(b.z, b.w, c.x);
                } else {
                    const float4* tp = tris + 3 * (size_t)(leaf_off + i);
                    float4 a = ldg4_stream(tp), b = ldg4_stream(tp + 1);
                    c = ldg4_stream(tp + 2);
                    p0 = mk3(a.x, a.y, a.z); p1 = mk3(a.w, b.x, b.y); p2 = mk3(b.z, b.w, c.x);
                }
                if (INST && (__float_as_uint(c.w) & TRI_INSTANCE)) {
                    // TransformedPrimitive::intersect / intersect_p: go into the object's tree with the object-space ray
                    const uint32_t id = __float_as_uint(p0.x);
                    const DInstance& I = sc.instances[id];
                    PB_PUSH(leaf_off + i + 1);
                    PB_PUSH(leaf_n - i - 1);
                    PB_PUSH(PB_SENTINEL);
                    t_max_w = t_max;
                    inst_hit = false;
                    cur_inst = (int)id;
                    PB_SAVE_WORLD();
                    V3 oo, od;
                    float tm = t_max;
                    xf_ray_dev(I.m_inv, r.o, r.d, tm, oo, od);
                    r = make_ray(oo, od);
                    t_max = tm;
                    cur = I.root;
                    leaf_n = 0;
                    entered = true;
                    break;
                }
                THit h;
                if (COUNT) wc.tris++;
                if (tri_test(p0, p1, p2, r, t_max, h) &&
                    !(ALPHA && (__float_as_uint(c.w) & (any_hit ? (uint32_t)(TRI_ALPHA | TRI_SHADOW_ALPHA) : (uint32_t)TRI_ALPHA)) &&
                      alpha_rejects(sc, leaf_off + i, p0, p1, p2, h.b0, h.b1, h.b2, __float_as_uint(c.w), any_hit))) {
                    t_max = h.t;
                    best = h;
                    best_prim = (int)(leaf_off + i);
                    if (INST) {
                        best_inst = cur_inst;
                        if (cur_inst >= 0) inst_hit = true; else hit_flag = true;
                    }
                    if (any_hit) { done = true; break; }
                }
            }
            if (!entered) {
                leaf_n = 0;
                if (!done) PB_NEXT();
            }
        }
        // ---- retire finished rays ------------------------------------------------------------------
        if (active && done) {
            // INST, closest hit: the reference reports a hit only when some primitive RETURNED true (an identity instance does not,
            // although it overwrote the interaction and shortened the ray)
            if (INST && !any_hit && !hit_flag) best_prim = -1;
            if (MODE == 0) {
                uint32_t slot = dest & PB_RAY_SLOT_MASK, kind = dest >> 30;
                if (kind == RAY_SHADOW) io.occl[slot] = best_prim >= 0 ? 1u : 0u;
                else {
                    float4 rec = make_float4(__int_as_float(best_prim), best.b0, best.b1, best.b2);
                    if (kind == RAY_EXTEND) { io.hit[slot] = rec; if (INST) io.hit_inst[slot] = (uint32_t)best_inst; }
                    else { io.mis_hit[slot] = rec; if (INST) io.mis_inst[slot] = (uint32_t)best_inst; }
                }
            } else if (MODE == 1) {
                io.out_prim[ray_id] = best_prim;
                io.out_t[ray_id] = best_prim >= 0 ? (INST ? t_max : best.t) : 0.0f;
                io.out_b[3 * (size_t)ray_id] = best_prim >= 0 ? best.b0 : 0.0f;
                io.out_b[3 * (size_t)ray_id + 1] = best_prim >= 0 ? best.b1 : 0.0f;
                io.out_b[3 * (size_t)ray_id + 2] = best_prim >= 0 ? best.b2 : 0.0f;
            } else io.out_occ[ray_id] = best_prim >= 0 ? 1 : 0;
            active = false;
        }
    }
    (void)inf;
    uint32_t a = n_closest, b = n_shadow;
    for (int o = 16; o > 0; o >>= 1) { a += __shfl_xor_sync(FULL, a, o); b += __shfl_xor_sync(FULL, b, o); }
    if (lane == 0) {
        if (a) atomicAdd(&cnt->closest_rays, (unsigned long long)a);
        if (b) atomicAdd(&cnt->shadow_rays, (unsigned long long)b);
    }
    if (COUNT) {
        uint32_t c = wc.nodes, e = wc.tris;
        for (int o = 16; o > 0; o >>= 1) { c += __shfl_xor_sync(FULL, c, o); e += __shfl_xor_sync(FULL, e, o); }
        if (lane == 0) { atomicAdd(&cnt->nodes_visited, (unsigned long long)c); atomicAdd(&cnt->tris_tested, (unsigned long long)e); }
    }
}

// -----------------------------------------------------------------------------------------------
// Wide-record traversal (MODE 0, no instances, no alpha masks, scene in global memory): the same rays, the same visit order and the
// same accepted hits as trace_rays, from a node array re-laid for the GPU (k_wide_build): one 64-byte record per INTERIOR node
// holding BOTH children's boxes, {c0.pmin.xyz, c0.pmax.x} {c0.pmax.yz, c1.pmin.xy} {c1.pmin.z, c1.pmax.xyz} {ref0, ref1, axis, -}
// with ref = record index of an interior child, or first primitive | n_prims << 28 of a leaf child.  A visit fetches one record
// (one dependent memory round trip per tree level instead of two) and tests both boxes in one instruction stream.  The reference
// tests a far child's box only when it pops it, against the t_max of that moment; slab_test depends on t_max through its last
// comparison alone, so the far child's entry parameter travels on the stack and that comparison is made at the pop (slab_geo).
#ifndef PB_WIDE_STACK_ENTRIES
#define PB_WIDE_STACK_ENTRIES 16  // two words per entry: the shared-memory budget of the 32-entry narrow stack
#endif
#define PB_WIDE_LEAF_SHIFT 28
// PB_TRACE_PHASE_CLOCKS (diagnostic builds only, tools/build_variants.py): lane 0 of every trace_rays_wide warp sums the clock64() cycles
// of the ray refill, the node phase and the leaf phase (the retire stores fall outside all three), and counts the rounds in which some lane
// held a leaf; every lane counts its triangle tests.  render_impl prints and clears the totals after each render.
#ifdef PB_TRACE_PHASE_CLOCKS
__device__ unsigned long long g_trace_phase[5];  // refill, node, leaf cycles; leaf rounds; triangle tests
#define PB_PHASE_DECL() unsigned long long ph_[5] = {0, 0, 0, 0, 0}; long long ph_t = clock64()
#define PB_PHASE_START() (ph_t = clock64())
#define PB_PHASE_LAP(i) do { const long long n_ = clock64(); ph_[i] += (unsigned long long)(n_ - ph_t); ph_t = n_; } while (0)
#define PB_PHASE_COUNT(i, n) (ph_[i] += (n))
#define PB_PHASE_FLUSH()                                                                                        \
    do {                                                                                                        \
        if (lane == 0) for (int i_ = 0; i_ < 4; ++i_) atomicAdd(&g_trace_phase[i_], ph_[i_]);                   \
        if (ph_[4]) atomicAdd(&g_trace_phase[4], ph_[4]);                                                       \
    } while (0)
#else
#define PB_PHASE_DECL() do {} while (0)
#define PB_PHASE_START() do {} while (0)
#define PB_PHASE_LAP(i) do {} while (0)
#define PB_PHASE_COUNT(i, n) do {} while (0)
#define PB_PHASE_FLUSH() do {} while (0)
#endif
template <bool INST>
PB_D void trace_rays_wide(const DScene& sc, const float4* __restrict__ wide, const float4* __restrict__ tris, const TraceIO& io, uint32_t n_rays,
                          uint32_t* __restrict__ cursor, DCounters* cnt, int walk_steps) {
    const unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    constexpr int NS = PB_WIDE_STACK_ENTRIES;
    constexpr int NL = (INST ? 136 : 64) - NS;  // INST: the world tree's 64 + the object's 64 + resume / sentinel entries
    __shared__ uint32_t s_ref[NS][PB_TRACE_THREADS_];
    __shared__ float s_tmin[NS][PB_TRACE_THREADS_];
    // INST: the world ray's traversal constants while the lane is inside an instance (see trace_rays)
    __shared__ float s_world[INST ? 13 : 1][PB_TRACE_THREADS_];
    uint32_t l_ref[NL];
    float l_tmin[NL];
    RayPre r;
    float t_max = 0.0f;
    THit best;
    int best_prim = -1;
    uint32_t sp = 0, cur = 0, dest = 0, leaf_off = 0, leaf_n = 0;
    bool active = false, any_hit = false, exhausted = n_rays == 0;
    // INST state, as in trace_rays: the instance being traversed, whether it produced a candidate, the world ray's t_max while inside
    int cur_inst = -1, best_inst = -1;
    bool inst_hit = false, hit_flag = false;
    float t_max_w = 0.0f;
    uint32_t n_closest = 0, n_shadow = 0;
    const float neg_inf = __int_as_float((int)0xff800000);
#define PB_WPUSH(ref_, tmin_)                                                                                   \
    do {                                                                                                        \
        if (sp < (uint32_t)NS) { s_ref[sp][threadIdx.x] = (ref_); s_tmin[sp][threadIdx.x] = (tmin_); }           \
        else { l_ref[sp - NS] = (ref_); l_tmin[sp - NS] = (tmin_); }                                            \
        ++sp;                                                                                                   \
    } while (0)
    // next pending subtree whose entry parameter is still below t_max (the reference's box test at the pop), or none left.  INST: the
    // sentinel ends an instance -- TransformedPrimitive::intersect's epilogue, the world ray comes back -- and the entry below it (if
    // any) resumes the interrupted world leaf (its entry parameter is -inf: the reference does not test that leaf's box again)
#define PB_WPOP()                                                                                               \
    do {                                                                                                        \
        for (;;) {                                                                                              \
            if (sp == 0u) { done = true; break; }                                                               \
            --sp;                                                                                               \
            const uint32_t e_ = sp < (uint32_t)NS ? s_ref[sp][threadIdx.x] : l_ref[sp - NS];                    \
            const float m_ = sp < (uint32_t)NS ? s_tmin[sp][threadIdx.x] : l_tmin[sp - NS];                     \
            if (INST && e_ == PB_SENTINEL) {                                                                    \
                if (inst_hit) {                                                                                 \
                    t_max_w = t_max; /* r.t_max.set(ray.t_max.get()): the OBJECT ray's parameter, as written */ \
                    if (io.instancing == 1u || !sc.instances[cur_inst].identity) hit_flag = true;               \
                }                                                                                               \
                {                                                                                               \
                    const int t_ = threadIdx.x;                                                                 \
                    r = unpack_ray(mk3(s_world[0][t_], s_world[INST ? 1 : 0][t_], s_world[INST ? 2 : 0][t_]),    \
                                   mk3(s_world[INST ? 3 : 0][t_], s_world[INST ? 4 : 0][t_], s_world[INST ? 5 : 0][t_]), \
                                   make_float4(s_world[INST ? 6 : 0][t_], s_world[INST ? 7 : 0][t_], s_world[INST ? 8 : 0][t_], s_world[INST ? 12 : 0][t_]), \
                                   make_float4(s_world[INST ? 9 : 0][t_], s_world[INST ? 10 : 0][t_], s_world[INST ? 11 : 0][t_], 0.0f)); \
                }                                                                                               \
                t_max = t_max_w;                                                                                \
                cur_inst = -1;                                                                                  \
                continue;                                                                                       \
            }                                                                                                   \
            if (m_ < t_max) { nxt = e_; break; }                                                                \
        }                                                                                                       \
    } while (0)
#define PB_WGOTO()                                                                                              \
    do {                                                                                                        \
        if (!done) {                                                                                            \
            if (nxt >> PB_WIDE_LEAF_SHIFT) { leaf_n = nxt >> PB_WIDE_LEAF_SHIFT; leaf_off = nxt & ((1u << PB_WIDE_LEAF_SHIFT) - 1u); } \
            else cur = nxt;                                                                                     \
        }                                                                                                       \
    } while (0)
    PB_PHASE_DECL();
    for (;;) {
        PB_PHASE_START();
        unsigned idle = __ballot_sync(FULL, !active);
        bool done = false;
        if (idle && !exhausted) {
            uint32_t base = 0;
            if (lane == 0) base = atomicAdd(cursor, (uint32_t)__popc(idle));
            base = __shfl_sync(FULL, base, 0);
            if (base >= n_rays) exhausted = true;
            const uint32_t my = base + (uint32_t)__popc(idle & ((1u << lane) - 1u));
            if (!active && my < n_rays) {
                const uint32_t qi = io.perm ? __ldg(io.perm + my) : my;
                const float4 a = ldg4_stream(io.rays + 2 * (size_t)qi), b = ldg4_stream(io.rays + 2 * (size_t)qi + 1);
                t_max = a.w;
                dest = __float_as_uint(b.w);
                any_hit = (dest >> 30) == RAY_SHADOW;
                r = make_ray(mk3(a.x, a.y, a.z), mk3(b.x, b.y, b.z));
                best_prim = -1;
                best.t = 0.0f; best.b0 = best.b1 = best.b2 = 0.0f;
                sp = 0; cur = 0; leaf_n = 0;
                cur_inst = -1; best_inst = -1; inst_hit = false; hit_flag = false;
                active = true;
                if (any_hit) n_shadow++; else n_closest++;
                // the root's own box (the only box that is not some record's child), bvh.rs:421-424
                const float4 n0 = ldg4_keep(sc.nodes), n1 = ldg4_keep(sc.nodes + 1);
                done = !slab_test(n0, n1, r, t_max);
            }
        }
        if (!__any_sync(FULL, active)) break;
        PB_PHASE_LAP(0);
        // ---- node phase ---------------------------------------------------------------------------
        for (int step = 0; step < walk_steps; ++step) {  // record visits per lane and round (each covers two tree levels)
            if (!(active && !done && leaf_n == 0u)) break;
            const float4* rec = wide + 4 * (size_t)cur;
            const float4 f0 = ldg4_keep(rec), f1 = ldg4_keep(rec + 1), f2 = ldg4_keep(rec + 2), f3 = ldg4_keep(rec + 3);
            float tm0, tm1;
            const bool h0 = slab_geo(f0.x, f0.y, f0.z, f0.w, f1.x, f1.y, r, tm0) && tm0 < t_max;
            const bool h1 = slab_geo(f1.z, f1.w, f2.x, f2.y, f2.z, f2.w, r, tm1) && tm1 < t_max;
            const bool neg = ((r.negmask >> (__float_as_uint(f3.z) & 3u)) & 1u) != 0u;  // near child first (bvh.rs:446-453)
            const uint32_t ref0 = __float_as_uint(f3.x), ref1 = __float_as_uint(f3.y);
            const uint32_t ref_n = neg ? ref1 : ref0, ref_f = neg ? ref0 : ref1;
            const bool hn = neg ? h1 : h0, hf = neg ? h0 : h1;
            const float tf = neg ? tm0 : tm1;
            if (hn && hf) PB_WPUSH(ref_f, tf);
            uint32_t nxt = hn ? ref_n : ref_f;
            if (!hn && !hf) PB_WPOP();
            PB_WGOTO();
        }
        PB_PHASE_LAP(1);
#ifdef PB_TRACE_PHASE_CLOCKS
        if (__any_sync(FULL, active && leaf_n)) PB_PHASE_COUNT(3, 1);
#endif
        // ---- leaf phase ----------------------------------------------------------------------------
        if (active && leaf_n) {
            bool entered = false;
            for (uint32_t i = 0; i < leaf_n; ++i) {
                // Plain scenes load triangles through L1 (no L1::no_allocate): on the H100 that made k_trace 3-4 % shorter on both the
                // statue and the conference scene (DESIGN.md §7) -- rays traced close together test the same leaves.  The instanced kernel
                // keeps the streaming hint; it was not measured without it.
                const float4* tp = tris + 3 * (size_t)(leaf_off + i);
                const float4 a = INST ? ldg4_stream(tp) : __ldg(tp), b = INST ? ldg4_stream(tp + 1) : __ldg(tp + 1), c = INST ? ldg4_stream(tp + 2) : __ldg(tp + 2);
                if (INST && (__float_as_uint(c.w) & TRI_INSTANCE)) {
                    // TransformedPrimitive::intersect / intersect_p (primitive.rs:216-261): the rest of this leaf waits on the stack
                    // under a sentinel, the ray goes into the object's tree in object space
                    const uint32_t id = __float_as_uint(a.x);
                    const DInstance& I = sc.instances[id];
                    if (leaf_n - i - 1u) PB_WPUSH((leaf_off + i + 1u) | ((leaf_n - i - 1u) << PB_WIDE_LEAF_SHIFT), neg_inf);
                    PB_WPUSH(PB_SENTINEL, neg_inf);
                    t_max_w = t_max;
                    inst_hit = false;
                    cur_inst = (int)id;
                    {
                        const int t_ = threadIdx.x;
                        s_world[0][t_] = r.o.x; s_world[INST ? 1 : 0][t_] = r.o.y; s_world[INST ? 2 : 0][t_] = r.o.z;
                        s_world[INST ? 3 : 0][t_] = r.d.x; s_world[INST ? 4 : 0][t_] = r.d.y; s_world[INST ? 5 : 0][t_] = r.d.z;
                        s_world[INST ? 6 : 0][t_] = r.inv_dir.x; s_world[INST ? 7 : 0][t_] = r.inv_dir.y; s_world[INST ? 8 : 0][t_] = r.inv_dir.z;
                        s_world[INST ? 9 : 0][t_] = r.sx; s_world[INST ? 10 : 0][t_] = r.sy; s_world[INST ? 11 : 0][t_] = r.sz;
                        s_world[INST ? 12 : 0][t_] = __uint_as_float((uint32_t)r.kz | (r.negmask << 2));
                    }
                    V3 oo, od;
                    float tm = t_max;
                    xf_ray_dev(I.m_inv, r.o, r.d, tm, oo, od);
                    r = make_ray(oo, od);
                    t_max = tm;
                    // the object tree's root: its own box first (BVHAccel::intersect of the object), then its record -- or, for a
                    // one-node tree, its primitives
                    const float4 n0 = ldg4_keep(sc.nodes + 2 * (size_t)I.root), n1 = ldg4_keep(sc.nodes + 2 * (size_t)I.root + 1);
                    leaf_n = 0;
                    entered = true;
                    if (slab_test(n0, n1, r, t_max)) {
                        const uint32_t meta = __float_as_uint(n1.w);
                        if (meta & 0xffffu) { leaf_off = __float_as_uint(n1.z); leaf_n = meta & 0xffffu; }  // (a leaf root: tested next round)
                        else cur = I.root;
                    } else {
                        uint32_t nxt = 0;
                        PB_WPOP();  // pops the sentinel at once: back to the world
                        PB_WGOTO();
                    }
                    break;
                }
                THit h;
                PB_PHASE_COUNT(4, 1);
                if (tri_test(mk3(a.x, a.y, a.z), mk3(a.w, b.x, b.y), mk3(b.z, b.w, c.x), r, t_max, h)) {
                    t_max = h.t;
                    best = h;
                    best_prim = (int)(leaf_off + i);
                    if (INST) {
                        best_inst = cur_inst;
                        if (cur_inst >= 0) inst_hit = true; else hit_flag = true;
                    }
                    if (any_hit) { done = true; break; }
                }
            }
            if (!entered) {
                leaf_n = 0;
                if (!done) {
                    uint32_t nxt = 0;
                    PB_WPOP();
                    PB_WGOTO();
                }
            }
        }
        PB_PHASE_LAP(2);
        // ---- retire ----------------------------------------------------------------------------------
        if (active && done) {
            // INST, closest hit: the reference reports a hit only when some primitive RETURNED true (an identity instance does not)
            if (INST && !any_hit && !hit_flag) best_prim = -1;
            const uint32_t slot = dest & PB_RAY_SLOT_MASK, kind = dest >> 30;
            if (kind == RAY_SHADOW) io.occl[slot] = best_prim >= 0 ? 1u : 0u;
            else {
                const float4 rec = make_float4(__int_as_float(best_prim), best.b0, best.b1, best.b2);
                if (kind == RAY_EXTEND) { io.hit[slot] = rec; if (INST) io.hit_inst[slot] = (uint32_t)best_inst; }
                else { io.mis_hit[slot] = rec; if (INST) io.mis_inst[slot] = (uint32_t)best_inst; }
            }
            active = false;
        }
    }
#undef PB_WPOP
#undef PB_WGOTO
#undef PB_WPUSH
    PB_PHASE_FLUSH();
    uint32_t a = n_closest, b = n_shadow;
    for (int o = 16; o > 0; o >>= 1) { a += __shfl_xor_sync(FULL, a, o); b += __shfl_xor_sync(FULL, b, o); }
    if (lane == 0) {
        if (a) atomicAdd(&cnt->closest_rays, (unsigned long long)a);
        if (b) atomicAdd(&cnt->shadow_rays, (unsigned long long)b);
    }
}

// -----------------------------------------------------------------------------------------------
// trace_rays_wide with ONE LEAF OF LOOK-AHEAD per lane (PB_WIDE_SPEC=1; scenes without instances).  In the plain wide walk a lane
// that reaches a leaf idles until the node phase of its warp is over; here it remembers the leaf and keeps walking -- with the t_max it
// has, which the remembered leaf may yet shorten -- until it meets a second leaf.  Nothing the reference decides changes: every
// pending subtree, the node being expanded and the second leaf all carry their entry parameter t_min, and each is compared with the
// t_max of the moment the reference would have looked at it (after the first leaf's triangles): what the stale t_max let through too
// generously is dropped then.  Child boxes lie inside their parent's, so t_min never decreases down the tree and a dropped node's
// descendants drop as well; the stack order, and with it the order in which leaves are tested, is the reference's.
PB_D void trace_rays_wide_spec(const DScene& sc, const float4* __restrict__ wide, const float4* __restrict__ tris, const TraceIO& io, uint32_t n_rays,
                               uint32_t* __restrict__ cursor, DCounters* cnt, int walk_steps) {
    const unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    constexpr int NS = PB_WIDE_STACK_ENTRIES;
    __shared__ uint32_t s_ref[NS][PB_TRACE_THREADS_];
    __shared__ float s_tmin[NS][PB_TRACE_THREADS_];
    uint32_t l_ref[64 - NS];
    float l_tmin[64 - NS];
    RayPre r;
    float t_max = 0.0f, cur_tmin = 0.0f, leaf2_tmin = 0.0f;
    THit best;
    int best_prim = -1;
    uint32_t sp = 0, cur = 0, dest = 0, leaf1 = 0, leaf2 = 0;  // leaf references: first primitive | count << 28, 0 = none
    bool active = false, any_hit = false, exhausted = n_rays == 0, have_cur = false;
    uint32_t n_closest = 0, n_shadow = 0;
    const float neg_inf = __int_as_float((int)0xff800000);
#define PB_SPOP()                                                                                               \
    do {                                                                                                        \
        found = false;                                                                                          \
        while (sp != 0u) {                                                                                      \
            --sp;                                                                                               \
            const uint32_t e_ = sp < (uint32_t)NS ? s_ref[sp][threadIdx.x] : l_ref[sp - NS];                    \
            const float m_ = sp < (uint32_t)NS ? s_tmin[sp][threadIdx.x] : l_tmin[sp - NS];                     \
            if (m_ < t_max) { nxt = e_; tm = m_; found = true; break; }                                         \
        }                                                                                                       \
    } while (0)
    // where the walk goes with what it found: an interior record to expand; the first leaf, which is remembered while the walk goes
    // on; the second leaf, which stops it; or nothing left
#define PB_SROUTE()                                                                                             \
    do {                                                                                                        \
        for (;;) {                                                                                              \
            if (!found) { have_cur = false; break; }                                                            \
            if (!(nxt >> PB_WIDE_LEAF_SHIFT)) { cur = nxt; cur_tmin = tm; have_cur = true; break; }             \
            if (!leaf1) { leaf1 = nxt; PB_SPOP(); continue; }                                                   \
            leaf2 = nxt; leaf2_tmin = tm; have_cur = false; break;                                              \
        }                                                                                                       \
    } while (0)
    for (;;) {
        unsigned idle = __ballot_sync(FULL, !active);
        bool done = false;
        if (idle && !exhausted) {
            uint32_t base = 0;
            if (lane == 0) base = atomicAdd(cursor, (uint32_t)__popc(idle));
            base = __shfl_sync(FULL, base, 0);
            if (base >= n_rays) exhausted = true;
            const uint32_t my = base + (uint32_t)__popc(idle & ((1u << lane) - 1u));
            if (!active && my < n_rays) {
                const uint32_t qi = io.perm ? __ldg(io.perm + my) : my;
                const float4 a = ldg4_stream(io.rays + 2 * (size_t)qi), b = ldg4_stream(io.rays + 2 * (size_t)qi + 1);
                t_max = a.w;
                dest = __float_as_uint(b.w);
                any_hit = (dest >> 30) == RAY_SHADOW;
                r = make_ray(mk3(a.x, a.y, a.z), mk3(b.x, b.y, b.z));
                best_prim = -1;
                best.t = 0.0f; best.b0 = best.b1 = best.b2 = 0.0f;
                sp = 0; cur = 0; cur_tmin = neg_inf; leaf1 = 0; leaf2 = 0;
                active = true;
                if (any_hit) n_shadow++; else n_closest++;
                const float4 n0 = ldg4_keep(sc.nodes), n1 = ldg4_keep(sc.nodes + 1);  // the root's own box (bvh.rs:421-424)
                have_cur = slab_test(n0, n1, r, t_max);
            }
        }
        if (!__any_sync(FULL, active)) break;
        // ---- node phase ---------------------------------------------------------------------------
        for (int step = 0; step < walk_steps; ++step) {
            if (!(active && have_cur)) break;
            const float4* rec = wide + 4 * (size_t)cur;
            const float4 f0 = ldg4_keep(rec), f1 = ldg4_keep(rec + 1), f2 = ldg4_keep(rec + 2), f3 = ldg4_keep(rec + 3);
            float tm0, tm1;
            const bool h0 = slab_geo(f0.x, f0.y, f0.z, f0.w, f1.x, f1.y, r, tm0) && tm0 < t_max;
            const bool h1 = slab_geo(f1.z, f1.w, f2.x, f2.y, f2.z, f2.w, r, tm1) && tm1 < t_max;
            const bool neg = ((r.negmask >> (__float_as_uint(f3.z) & 3u)) & 1u) != 0u;
            const uint32_t ref0 = __float_as_uint(f3.x), ref1 = __float_as_uint(f3.y);
            const uint32_t ref_n = neg ? ref1 : ref0, ref_f = neg ? ref0 : ref1;
            const bool hn = neg ? h1 : h0, hf = neg ? h0 : h1;
            const float tn = neg ? tm1 : tm0, tf = neg ? tm0 : tm1;
            if (hn && hf) {
                if (sp < (uint32_t)NS) { s_ref[sp][threadIdx.x] = ref_f; s_tmin[sp][threadIdx.x] = tf; }
                else { l_ref[sp - NS] = ref_f; l_tmin[sp - NS] = tf; }
                ++sp;
            }
            uint32_t nxt = hn ? ref_n : ref_f;
            float tm = hn ? tn : tf;
            bool found = hn || hf;
            if (!found) PB_SPOP();
            PB_SROUTE();
        }
        // ---- leaf phase: the first pending leaf of every lane; then the look-ahead is held against the t_max that leaf left ----
        if (active && leaf1) {
            const uint32_t leaf_n = leaf1 >> PB_WIDE_LEAF_SHIFT, leaf_off = leaf1 & ((1u << PB_WIDE_LEAF_SHIFT) - 1u);
            for (uint32_t i = 0; i < leaf_n; ++i) {
                const float4* tp = tris + 3 * (size_t)(leaf_off + i);
                const float4 a = ldg4_stream(tp), b = ldg4_stream(tp + 1), c = ldg4_stream(tp + 2);
                THit h;
                if (tri_test(mk3(a.x, a.y, a.z), mk3(a.w, b.x, b.y), mk3(b.z, b.w, c.x), r, t_max, h)) {
                    t_max = h.t;
                    best = h;
                    best_prim = (int)(leaf_off + i);
                    if (any_hit) { done = true; break; }
                }
            }
            leaf1 = 0;
            if (!done) {
                bool resume = false;
                if (leaf2) {  // the walk stopped at a second leaf: it is next if the reference would still visit it, and the walk resumes
                    if (leaf2_tmin < t_max) leaf1 = leaf2;
                    leaf2 = 0;
                    resume = true;
                } else if (have_cur && !(cur_tmin < t_max)) { have_cur = false; resume = true; }  // the record being expanded was reached too generously
                if (resume) {
                    uint32_t nxt = 0;
                    float tm = 0.0f;
                    bool found;
                    PB_SPOP();
                    PB_SROUTE();
                }
            }
        }
        if (active && !done && !leaf1 && !leaf2 && !have_cur) done = true;  // nothing pending: BVHAccel::intersect's loop has ended
        // ---- retire ----------------------------------------------------------------------------------
        if (active && done) {
            const uint32_t slot = dest & PB_RAY_SLOT_MASK, kind = dest >> 30;
            if (kind == RAY_SHADOW) io.occl[slot] = best_prim >= 0 ? 1u : 0u;
            else {
                const float4 rec = make_float4(__int_as_float(best_prim), best.b0, best.b1, best.b2);
                if (kind == RAY_EXTEND) io.hit[slot] = rec; else io.mis_hit[slot] = rec;
            }
            active = false;
        }
    }
#undef PB_SPOP
#undef PB_SROUTE
    uint32_t a = n_closest, b = n_shadow;
    for (int o = 16; o > 0; o >>= 1) { a += __shfl_xor_sync(FULL, a, o); b += __shfl_xor_sync(FULL, b, o); }
    if (lane == 0) {
        if (a) atomicAdd(&cnt->closest_rays, (unsigned long long)a);
        if (b) atomicAdd(&cnt->shadow_rays, (unsigned long long)b);
    }
}

}  // namespace pb
