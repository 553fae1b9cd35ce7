// pb_interaction.cuh -- SurfaceInteraction reconstruction and area-light sampling on the device.
//   Triangle::intersect, interaction part     src/shapes/triangle.rs:274-448
//   Triangle::sample / sample_with_ref_point   src/shapes/triangle.rs:676-744
//   Triangle::pdf_with_ref_point               src/shapes/triangle.rs:745-764
//   DiffuseAreaLight::sample_li / l            src/lights/diffuse.rs:64-84,164-170
//   InteractionCommon::spawn_ray / spawn_ray_to  src/core/interaction.rs:58-94
// The reference fills a SurfaceInteraction for every accepted BVH candidate; only the last one
// survives, so the wavefront stores (prim, b0, b1, b2) and rebuilds the interaction once here.
// compute_differentials (interaction.rs:388-474) only feeds texture filtering; with constant
// textures it cannot influence the result and is not evaluated.
#pragma once
#include "pb_trace.cuh"

namespace pb {

struct Isect {
    V3 p, p_error, n;      // InteractionCommon (wo = -ray.d is kept by the caller)
    V3 ns;                 // shading.n
    V3 sh_dpdu;            // shading.dpdu
    V3 dpdu;               // isect.dpdu (the geometric one; AOIntegrator builds its frame from it)
    V3 dpdv;               // isect.dpdv and isect.uv: read by k_texture only (compute_differentials, UVMapping2D)
    float2 uv;
    V3 sh_dpdv, sh_dndu, sh_dndv;  // shading.dpdv / dndu / dndv (triangle.rs:384-421): read by k_texture only (Material::bump)
    bool shape_flips;      // isect.shape is Some and reverse_orientation ^ transform_swaps_handedness (set_shading_geometry)
    uint32_t material;
    int area_light;
};

struct TriData {
    V3 p0, p1, p2;
    uint32_t material, flags;
    int area_light;
};
PB_D TriData load_tri_full(const DScene& sc, uint32_t prim) {
    float4 a = __ldg(sc.tri_verts + 3 * (size_t)prim), b = __ldg(sc.tri_verts + 3 * (size_t)prim + 1), c = __ldg(sc.tri_verts + 3 * (size_t)prim + 2);
    TriData t;
    t.p0 = mk3(a.x, a.y, a.z);
    t.p1 = mk3(a.w, b.x, b.y);
    t.p2 = mk3(b.z, b.w, c.x);
    t.material = __float_as_uint(c.y);
    t.area_light = (int)__float_as_uint(c.z);
    t.flags = __float_as_uint(c.w);
    return t;
}
PB_D V3 ld3(const float* __restrict__ a, uint32_t i) { return mk3(__ldg(a + 3 * (size_t)i), __ldg(a + 3 * (size_t)i + 1), __ldg(a + 3 * (size_t)i + 2)); }

PB_D Isect tri_interaction(const DScene& sc, uint32_t prim, float b0, float b1, float b2) {
    TriData t = load_tri_full(sc, prim);
    const V3 p0 = t.p0, p1 = t.p1, p2 = t.p2;
    uint4 idx = make_uint4(0, 0, 0, 0);
    if (t.flags & (TRI_HAS_N | TRI_HAS_UV | TRI_HAS_S)) idx = __ldg(sc.tri_idx + prim);
    float2 uv0 = make_float2(0.0f, 0.0f), uv1 = make_float2(1.0f, 0.0f), uv2 = make_float2(1.0f, 1.0f);  // triangle.rs:96-110
    if (t.flags & TRI_HAS_UV) {
        uv0 = make_float2(__ldg(sc.vuv + 2 * (size_t)idx.x), __ldg(sc.vuv + 2 * (size_t)idx.x + 1));
        uv1 = make_float2(__ldg(sc.vuv + 2 * (size_t)idx.y), __ldg(sc.vuv + 2 * (size_t)idx.y + 1));
        uv2 = make_float2(__ldg(sc.vuv + 2 * (size_t)idx.z), __ldg(sc.vuv + 2 * (size_t)idx.z + 1));
    }
    float duv02x = uv0.x - uv2.x, duv02y = uv0.y - uv2.y, duv12x = uv1.x - uv2.x, duv12y = uv1.y - uv2.y;
    V3 dp02 = p0 - p2, dp12 = p1 - p2;
    float determinant = duv02x * duv12y - duv02y * duv12x;
    bool degenerate_uv = fabsf(determinant) < 1e-8f;
    V3 dpdu = mk3(0.0f, 0.0f, 0.0f), dpdv = mk3(0.0f, 0.0f, 0.0f);
    if (!degenerate_uv) {
        float invdet = 1.0f / determinant;
        dpdu = (dp02 * duv12y - dp12 * duv02y) * invdet;
        dpdv = (dp02 * -duv12x + dp12 * duv02x) * invdet;
    }
    if (degenerate_uv || len2(cross3(dpdu, dpdv)) == 0.0f) coordinate_system(norm3(cross3(p2 - p0, p1 - p0)), dpdu, dpdv);
    Isect I;
    I.p_error = mk3(fabsf(b0 * p0.x) + fabsf(b1 * p1.x) + fabsf(b2 * p2.x), fabsf(b0 * p0.y) + fabsf(b1 * p1.y) + fabsf(b2 * p2.y),
                    fabsf(b0 * p0.z) + fabsf(b1 * p1.z) + fabsf(b2 * p2.z)) * gamma_n(7);
    I.p = p0 * b0 + p1 * b1 + p2 * b2;
    V3 surface_normal = norm3(cross3(dp02, dp12));
    if (t.flags & TRI_FLIP) surface_normal = -surface_normal;
    I.ns = surface_normal;
    I.sh_dpdu = dpdu;
    I.sh_dpdv = dpdv;
    I.sh_dndu = I.sh_dndv = mk3(0.0f, 0.0f, 0.0f);
    I.shape_flips = (t.flags & TRI_FLIP) != 0;
    I.dpdu = dpdu;
    I.dpdv = dpdv;
    I.uv = make_float2(uv0.x * b0 + uv1.x * b1 + uv2.x * b2, uv0.y * b0 + uv1.y * b1 + uv2.y * b2);  // triangle.rs uv_hit
    if (t.flags & (TRI_HAS_N | TRI_HAS_S)) {
        V3 ns;
        if (t.flags & TRI_HAS_N) {
            ns = ld3(sc.vn, idx.x) * b0 + ld3(sc.vn, idx.y) * b1 + ld3(sc.vn, idx.z) * b2;
            if (len2(ns) > 0.0f) ns = norm3(ns);
            else ns = surface_normal;
        } else ns = surface_normal;
        V3 ss;
        if (t.flags & TRI_HAS_S) {
            ss = ld3(sc.vs, idx.x) * b0 + ld3(sc.vs, idx.y) * b1 + ld3(sc.vs, idx.z) * b2;
            if (len2(ss) > 0.0f) ss = norm3(ss);
            else ss = norm3(dpdu);
        } else ss = norm3(dpdu);
        V3 ts = cross3(ss, ns);
        if (len2(ts) > 0.0f) { ts = norm3(ts); ss = cross3(ts, ns); }
        else coordinate_system(ns, ss, ts);
        if ((t.flags & TRI_HAS_N) && !degenerate_uv) {  // dndu / dndv of the shading geometry (triangle.rs:392-411)
            const V3 dn1 = ld3(sc.vn, idx.x) - ld3(sc.vn, idx.z), dn2 = ld3(sc.vn, idx.y) - ld3(sc.vn, idx.z);
            const float inv_det = 1.0f / determinant;
            I.sh_dndu = (dn1 * duv12y - dn2 * duv02y) * inv_det;
            I.sh_dndv = (dn1 * -duv12x + dn2 * duv02x) * inv_det;
        }
        I.ns = norm3(cross3(ss, ts));
        surface_normal = faceforward3(surface_normal, I.ns);
        I.sh_dpdu = ss;
        I.sh_dpdv = ts;
    }
    I.n = surface_normal;
    I.material = t.material;
    I.area_light = t.area_light;
    return I;
}

// Transform::transform_surface_interaction (transform.rs:815-860) with instance_to_world, for what the path uses of it: p and its
// absolute error (transform_point_with_abs_error :709-760), n and shading.n through the inverse transpose (normalised), dpdu /
// shading.dpdu as vectors, shading.n face-forwarded to n.
PB_D void isect_to_world(const DInstance& I, Isect& is) {
    const float* m = I.m;
    const float* mi = I.m_inv;
    const float x = is.p.x, y = is.p.y, z = is.p.z;
    const V3 pe = is.p_error;
    const float g3 = gamma_n(3);
    const float xp = m[0] * x + m[1] * y + m[2] * z + m[3];
    const float yp = m[4] * x + m[5] * y + m[6] * z + m[7];
    const float zp = m[8] * x + m[9] * y + m[10] * z + m[11];
    const float wp = m[12] * x + m[13] * y + m[14] * z + m[15];
    is.p_error = mk3((g3 + 1.0f) * (fabsf(m[0]) * pe.x + fabsf(m[1]) * pe.y + fabsf(m[2]) * pe.z) + g3 * (fabsf(m[0] * x) + fabsf(m[1] * y) + fabsf(m[2] * z) + fabsf(m[3])),
                     (g3 + 1.0f) * (fabsf(m[4]) * pe.x + fabsf(m[5]) * pe.y + fabsf(m[6]) * pe.z) + g3 * (fabsf(m[4] * x) + fabsf(m[5] * y) + fabsf(m[6] * z) + fabsf(m[7])),
                     (g3 + 1.0f) * (fabsf(m[8]) * pe.x + fabsf(m[9]) * pe.y + fabsf(m[10]) * pe.z) + g3 * (fabsf(m[8] * x) + fabsf(m[9] * y) + fabsf(m[10] * z) + fabsf(m[11])));
    is.p = mk3(xp, yp, zp);
    if (wp != 1.0f) { const float inv = 1.0f / wp; is.p = mk3(inv * xp, inv * yp, inv * zp); }
    auto xn = [mi](V3 n) { return mk3(mi[0] * n.x + mi[4] * n.y + mi[8] * n.z, mi[1] * n.x + mi[5] * n.y + mi[9] * n.z, mi[2] * n.x + mi[6] * n.y + mi[10] * n.z); };
    auto xv = [m](V3 v) { return mk3(m[0] * v.x + m[1] * v.y + m[2] * v.z, m[4] * v.x + m[5] * v.y + m[6] * v.z, m[8] * v.x + m[9] * v.y + m[10] * v.z); };
    is.n = norm3(xn(is.n));
    is.dpdu = xv(is.dpdu);
    is.dpdv = xv(is.dpdv);
    is.ns = norm3(xn(is.ns));
    is.sh_dpdu = xv(is.sh_dpdu);
    is.sh_dpdv = xv(is.sh_dpdv);
    is.sh_dndu = xn(is.sh_dndu);
    is.sh_dndv = xn(is.sh_dndv);
    is.shape_flips = false;  // ret.shape = None (transform.rs:830)
    is.ns = faceforward3(is.ns, is.n);
}
// The interaction of a hit as Scene::intersect hands it to the integrator: for a hit inside an instance the object-space
// interaction goes through instance_to_world (not for an identity instance), and in PBRT_INSTANCING_REFERENCE a transformed
// interaction has lost its primitive -- no material, no area light (transform.rs:856, quirk Q7).
// `wo` comes back as isect.wo, which estimate_direct evaluates the BSDF with (integrator.rs:447-449; PathIntegrator itself uses -ray.d,
// path.rs:142): -ray.d as Triangle::intersect left it (quirk Q5), or, for a transformed interaction, the object ray's -d carried back
// through instance_to_world and normalised (transform.rs:828).
PB_D Isect hit_interaction(const DScene& sc, uint32_t instancing, uint32_t prim, float b0, float b1, float b2, uint32_t inst, V3 ray_d, V3& wo) {
    Isect is = tri_interaction(sc, prim, b0, b1, b2);
    wo = -ray_d;
    if (inst != 0xffffffffu) {
        const DInstance& I = sc.instances[inst];
        const float* mi = I.m_inv;
        // the object ray's direction (Transform::transform_ray with the inverse) and its -d: the interaction's wo in object space
        const V3 d_obj = mk3(mi[0] * ray_d.x + mi[1] * ray_d.y + mi[2] * ray_d.z, mi[4] * ray_d.x + mi[5] * ray_d.y + mi[6] * ray_d.z,
                             mi[8] * ray_d.x + mi[9] * ray_d.y + mi[10] * ray_d.z);
        wo = -d_obj;
        if (!I.identity) {
            const float* m = I.m;
            wo = norm3(mk3(m[0] * wo.x + m[1] * wo.y + m[2] * wo.z, m[4] * wo.x + m[5] * wo.y + m[6] * wo.z, m[8] * wo.x + m[9] * wo.y + m[10] * wo.z));
            isect_to_world(I, is);
            if (instancing == 0u) { is.material = 0xffffffffu; is.area_light = -1; }
        }
    }
    return is;
}

// Hit point, geometric normal (with the reference's flips) and area light of a hit -- all that Le evaluation and
// pdf_li need.  Without per-vertex normals / tangents the normal does not depend on dpdu/dpdv or the shading
// frame (triangle.rs:336-340), so that part of Triangle::intersect is skipped; otherwise the full interaction is
// built (the face-forwarding of triangle.rs:416-417 needs the shading normal).
PB_D void tri_point_normal(const DScene& sc, uint32_t prim, float b0, float b1, float b2, V3& p, V3& n, int& area_light) {
    TriData t = load_tri_full(sc, prim);
    if (t.flags & (TRI_HAS_N | TRI_HAS_S)) {
        Isect I = tri_interaction(sc, prim, b0, b1, b2);
        p = I.p; n = I.n; area_light = I.area_light;
        return;
    }
    p = t.p0 * b0 + t.p1 * b1 + t.p2 * b2;
    n = norm3(cross3(t.p0 - t.p2, t.p1 - t.p2));
    if (t.flags & TRI_FLIP) n = -n;
    area_light = t.area_light;
}

PB_D Sp light_L(const DLight& l, V3 n, V3 w) {  // DiffuseAreaLight::l
    return (l.two_sided || dot3(n, w) > 0.0f) ? mksp(l.L[0], l.L[1], l.L[2]) : sp1(0.0f);
}

struct LightSample { V3 p, p_error, n; };
// Triangle::sample_with_ref_point(iref.p, u): returns the sampled point, pdf w.r.t. solid angle
PB_D LightSample tri_sample_ref(const DScene& sc, uint32_t prim, V3 ref_p, float2 u, float& pdf) {
    TriData t = load_tri_full(sc, prim);
    const V3 p0 = t.p0, p1 = t.p1, p2 = t.p2;
    float su0 = sqrtf(u.x);
    float bx = 1.0f - su0, by = u.y * su0;
    float bz = 1.0f - bx - by;
    LightSample s;
    s.p = p0 * bx + p1 * by + p2 * bz;
    V3 c = cross3(p1 - p0, p2 - p0);
    s.n = norm3(c);
    if (t.flags & TRI_HAS_N) {
        uint4 idx = __ldg(sc.tri_idx + prim);
        V3 ns = ld3(sc.vn, idx.x) * bx + ld3(sc.vn, idx.y) * by + ld3(sc.vn, idx.z) * bz;
        s.n = faceforward3(s.n, ns);
    } else if (t.flags & TRI_FLIP) s.n = s.n * -1.0f;
    s.p_error = (abs3(p0 * bx) + abs3(p1 * by) + abs3(p2 * bz)) * gamma_n(6);
    float area = 0.5f * len3(c);
    pdf = 1.0f / area;
    V3 wi = s.p - ref_p;
    if (len2(wi) == 0.0f) pdf = 0.0f;
    else {
        wi = norm3(wi);
        pdf *= len2(ref_p - s.p) / absdot3(s.n, -wi);
        if (isinf(pdf)) pdf = 0.0f;
    }
    return s;
}
// SpotLight::falloff (lights/spot.rs)
PB_D float spot_falloff(const DLight& l, V3 w) {
    V3 wl = norm3(mk3(l.w2l[0] * w.x + l.w2l[1] * w.y + l.w2l[2] * w.z, l.w2l[3] * w.x + l.w2l[4] * w.y + l.w2l[5] * w.z,
                      l.w2l[6] * w.x + l.w2l[7] * w.y + l.w2l[8] * w.z));
    float cos_theta = wl.z;
    if (cos_theta < l.cos_total_width) return 0.0f;
    if (cos_theta >= l.cos_falloff_start) return 1.0f;
    float delta = (cos_theta - l.cos_total_width) / (l.cos_falloff_start - l.cos_total_width);
    return (delta * delta) * (delta * delta);
}
// ---- InfiniteAreaLight (lights/infinite.rs) ---------------------------------------------------------------------------
PB_D V3 rot3(const float* m, V3 v) {  // Transform::transform_vector, upper 3x3
    return mk3(m[0] * v.x + m[1] * v.y + m[2] * v.z, m[3] * v.x + m[4] * v.y + m[5] * v.z, m[6] * v.x + m[7] * v.y + m[8] * v.z);
}
PB_D Sp env_texel(const DEnv& e, int s, int t) {  // MipMap::texel, ImageWrap::Repeat on a power-of-two level
    float4 v = __ldg(e.texels + (size_t)((uint32_t)t & (uint32_t)(e.h - 1)) * e.w + ((uint32_t)s & (uint32_t)(e.w - 1)));
    return mksp(v.x, v.y, v.z);
}
PB_D Sp env_lookup(const DEnv& e, float sx, float sy) {  // lookup_pnt_flt(st, 0) == triangle(0, st)  mipmap.rs:233-240,323-336
    float s = sx * (float)e.w - 0.5f, t = sy * (float)e.h - 0.5f;
    float fs = floorf(s), ft = floorf(t);
    int s0 = f2i_sat(fs), t0 = f2i_sat(ft);
    float ds = s - (float)s0, dt = t - (float)t0;
    Sp tmp1 = env_texel(e, s0 + 1, t0 + 1) * (ds * dt);
    Sp tmp2 = env_texel(e, s0 + 1, t0) * (ds * (1.0f - dt));
    Sp tmp3 = env_texel(e, s0, t0 + 1) * ((1.0f - ds) * dt);
    Sp tmp4 = env_texel(e, s0, t0) * ((1.0f - ds) * (1.0f - dt));
    return tmp4 + tmp3 + tmp2 + tmp1;
}
// Distribution1D::sample_continuous (sampling.rs:53-102) over func[n] / cdf[n+1]
PB_D float dist1d_sample_continuous(const float* __restrict__ func, const float* __restrict__ cdf, float func_int, int n, float u, float& pdf, int& off) {
    int first = 0, len = n + 1;
    while (len > 0) {
        int half = len >> 1, middle = first + half;
        if (__ldg(cdf + middle) <= u) { first = middle + 1; len -= half + 1; }
        else len = half;
    }
    int offset = first - 1;
    offset = offset < 0 ? 0 : (offset > n - 1 ? n - 1 : offset);
    off = offset;
    float c0 = __ldg(cdf + offset), c1 = __ldg(cdf + offset + 1);
    float du = u - c0;
    if ((c1 - c0) > 0.0f) du /= c1 - c0;
    pdf = (func_int > 0.0f) ? __ldg(func + offset) / func_int : 0.0f;
    return ((float)offset + du) / (float)n;
}
PB_D float spherical_theta(V3 v) { return acos_rn(clampf(v.z, -1.0f, 1.0f)); }  // geometry.rs:1584-1596
PB_D float spherical_phi(V3 v) {
    float p = atan2_rn(v.y, v.x);
    return p < 0.0f ? p + 2.0f * PB_PI : p;
}
// InfiniteAreaLight::le for a ray direction that left the scene
PB_D Sp env_le(const DEnv& e, V3 ray_d) {
    V3 w = norm3(rot3(e.w2l, ray_d));
    return env_lookup(e, spherical_phi(w) * PB_INV_2_PI, spherical_theta(w) * PB_INV_PI);
}
// InfiniteAreaLight::pdf_li
PB_D float env_pdf_li(const DEnv& e, V3 w) {
    V3 wi = rot3(e.w2l, w);
    float theta = spherical_theta(wi), phi = spherical_phi(wi);
    float sin_theta = sin_rn(theta);
    if (sin_theta == 0.0f) return 0.0f;
    float px = phi * PB_INV_2_PI, py = theta * PB_INV_PI;
    int iu = f2i_sat(px * (float)e.nu), iv = f2i_sat(py * (float)e.nv);  // Distribution2D::pdf sampling.rs:184-197
    iu = iu < 0 ? 0 : (iu > e.nu - 1 ? e.nu - 1 : iu);
    iv = iv < 0 ? 0 : (iv > e.nv - 1 ? e.nv - 1 : iv);
    float map_pdf = __ldg(e.cond_func + (size_t)iv * e.nu + iu) / e.marg_int;
    return map_pdf / (2.0f * PB_PI * PB_PI * sin_theta);
}
// Light levels of the kernels that sample lights, fixed per scene at creation: 0 = DiffuseAreaLights only (the other kinds are compiled
// out), 1 = every kind but the image lights, 2 = with GonioPhotometricLight / ProjectionLight (their own instantiations, so the others
// keep their code).
template <int LIGHTS>
PB_D bool light_is_delta(const DLight& l) {  // point, spot, distant, goniometric, projection (light.rs:178-190)
    return LIGHTS >= 2 ? (l.kind - 1u < 3u || l.kind - 5u < 2u) : l.kind - 1u < 3u;
}
// Light::le (light.rs:84-94): zero for everything but an infinite light
PB_D Sp light_le(const DScene& sc, const DLight& l, V3 ray_d) {
    if (l.kind != 4u) return sp1(0.0f);
    return env_le(sc.envs[l.env], ray_d);
}

// GonioPhotometricLight::scale (goniometric.rs:233-248) or ProjectionLight::projection (projection.rs:339-360) of the world direction
// w: a level-0 bilinear lookup of the map (lookup_pnt_flt(st, 0)), or exactly 1 for a goniometric light without one.
PB_D Sp image_light_scale(const DLight& l, const DEnv& e, V3 w) {
    if (l.kind == 5u) {
        if (e.w == 0) return sp1(1.0f);
        const V3 wn = norm3(rot3(l.w2l, w));
        const V3 wp = mk3(wn.x, wn.z, wn.y);  // std::mem::swap(&mut wp.y, &mut wp.z)
        return env_lookup(e, spherical_phi(wp) * PB_INV_2_PI, spherical_theta(wp) * PB_INV_PI);
    }
    const V3 wl = rot3(l.w2l, w);  // not normalised
    if (wl.z < e.hither) return sp1(0.0f);
    const float* m = e.proj;  // Transform::transform_point: the homogeneous divide multiplies by 1 / wp
    float px = m[0] * wl.x + m[1] * wl.y + m[2] * wl.z + m[3];
    float py = m[4] * wl.x + m[5] * wl.y + m[6] * wl.z + m[7];
    const float pw = m[12] * wl.x + m[13] * wl.y + m[14] * wl.z + m[15];
    if (pw != 1.0f) { const float inv = 1.0f / pw; px = inv * px; py = inv * py; }
    if (!(px >= e.screen[0] && px <= e.screen[2] && py >= e.screen[1] && py <= e.screen[3])) return sp1(0.0f);  // pnt2_inside_bnd2f
    float sx = px - e.screen[0], sy = py - e.screen[1];  // Bounds2f::offset
    if (e.screen[2] > e.screen[0]) sx /= e.screen[2] - e.screen[0];
    if (e.screen[3] > e.screen[1]) sy /= e.screen[3] - e.screen[1];
    return env_lookup(e, sx, sy);
}

// Light::sample_li: DiffuseAreaLight (diffuse.rs:64-84), PointLight, SpotLight, DistantLight (lights/{point,spot,distant}.rs),
// GonioPhotometricLight and ProjectionLight (goniometric.rs:249-265, projection.rs:362-378) at light level 2.
// For the delta lights the sampled "interaction" is a bare point (n = p_error = 0).
template <int LIGHTS>
PB_D Sp light_sample_li(const DScene& sc, const DLight& l, V3 ref_p, float2 u, V3& wi, float& pdf, LightSample& ls) {
    constexpr bool AREA_ONLY = LIGHTS == 0;
    if (!AREA_ONLY && l.kind == 4u) {  // InfiniteAreaLight::sample_li
        const DEnv& e = sc.envs[l.env];
        ls.p_error = mk3(0.0f, 0.0f, 0.0f);
        ls.n = mk3(0.0f, 0.0f, 0.0f);
        ls.p = ref_p;
        float pdf_v = 0.0f, pdf_u = 0.0f;
        int v = 0, dummy = 0;
        float d1 = dist1d_sample_continuous(e.marg_func, e.marg_cdf, e.marg_int, e.nv, u.y, pdf_v, v);
        float d0 = dist1d_sample_continuous(e.cond_func + (size_t)v * e.nu, e.cond_cdf + (size_t)v * (e.nu + 1), __ldg(e.cond_int + v), e.nu, u.x, pdf_u, dummy);
        float map_pdf = pdf_u * pdf_v;
        if (map_pdf == 0.0f) { pdf = 0.0f; return sp1(0.0f); }
        float theta = d1 * PB_PI, phi = d0 * 2.0f * PB_PI;
        float cos_theta, sin_theta, sin_phi, cos_phi;
        sincos_rn(theta, sin_theta, cos_theta);
        sincos_rn(phi, sin_phi, cos_phi);
        wi = rot3(e.l2w, mk3(sin_theta * cos_phi, sin_theta * sin_phi, cos_theta));
        pdf = map_pdf / (2.0f * PB_PI * PB_PI * sin_theta);
        if (sin_theta == 0.0f) pdf = 0.0f;
        ls.p = ref_p + wi * (2.0f * sc.world_radius);
        return env_lookup(e, d0, d1);
    }
    if (!AREA_ONLY && l.kind != 0u) {
        ls.p_error = mk3(0.0f, 0.0f, 0.0f);
        ls.n = mk3(0.0f, 0.0f, 0.0f);
        pdf = 1.0f;
        const V3 lp = mk3(l.p[0], l.p[1], l.p[2]);
        const Sp I = mksp(l.L[0], l.L[1], l.L[2]);
        if (l.kind == 3u) {  // distant
            wi = lp;
            ls.p = ref_p + lp * (2.0f * sc.world_radius);
            return I;
        }
        wi = norm3(lp - ref_p);
        ls.p = lp;
        float d2 = len2(lp - ref_p);
        if (LIGHTS >= 2 && l.kind >= 5u) return I * image_light_scale(l, sc.envs[l.env], -wi) / d2;
        if (l.kind == 1u) return I / d2;
        return I * spot_falloff(l, -wi) / d2;
    }
    ls = tri_sample_ref(sc, l.tri, ref_p, u, pdf);
    if (pdf == 0.0f || len2(ls.p - ref_p) == 0.0f) { pdf = 0.0f; return sp1(0.0f); }
    wi = norm3(ls.p - ref_p);
    return light_L(l, ls.n, -wi);
}
// DiffuseAreaLight::pdf_li for the ray (o, wi) spawned from the shaded point ref_p
template <int LIGHTS>
PB_D float light_pdf_li(const DScene& sc, const DLight& l, V3 ref_p, V3 ray_o, V3 wi) {
    if (LIGHTS != 0 && l.kind == 4u) return env_pdf_li(sc.envs[l.env], wi);
    V3 p0, p1, p2;
    load_tri(sc.tri_verts, l.tri, p0, p1, p2);
    RayPre r = make_ray(ray_o, wi);
    THit h;
    if (!tri_test(p0, p1, p2, r, __int_as_float(0x7f800000), h)) return 0.0f;
    V3 lp, ln;
    int al;
    tri_point_normal(sc, l.tri, h.b0, h.b1, h.b2, lp, ln, al);
    float area = 0.5f * len3(cross3(p1 - p0, p2 - p0));  // Triangle::area triangle.rs:667-675
    float pdf = len2(ref_p - lp) / (absdot3(ln, -wi) * area);
    if (isinf(pdf)) pdf = 0.0f;
    return pdf;
}

PB_D float power_heuristic(float f_pdf, float g_pdf) {  // nf = ng = 1  sampling.rs:229-233
    float f = 1.0f * f_pdf, g = 1.0f * g_pdf;
    return (f * f) / (f * f + g * g);
}

}  // namespace pb
