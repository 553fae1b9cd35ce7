// pb_lens.cuh -- RealisticCamera::generate_ray_differential (src/cameras/realistic.rs:198-327,656-735) on the device: the film
// point, the exit-pupil sample, the trace through the lens system and the camera ray weight.  The lens system and its exit-pupil
// bounds arrive as the caller's RealisticCamera built them (PbrtRealisticLens): the library computes neither focus nor pupil.
#pragma once
#include "pb_math.cuh"

namespace pb {

#define PB_PUPIL_BINS 64  // RealisticCamera::new: n_samples (realistic.rs:101)

// k_raygen's trailing by-value argument for the realistic camera (and the known-answer hook's).  Everything a sample reads is here,
// so that the per-sample element loop reads the kernel's constant bank and no struct of the other kernels grows.
struct DLens {
    float4 el[PBRT_MAX_LENS_ELEMENTS];  // element_interfaces {curvature_radius, thickness, eta, aperture_radius}, metres, film side last
    float4 pupil[PB_PUPIL_BINS];        // exit_pupil_bounds {pmin.x, pmin.y, pmax.x, pmax.y}
    float2 ext_min, ext_max;            // Film::get_physical_extent (film.rs:293-307), made on the host in the reference's f32 order
    float2 full_res;                    // Film.full_resolution
    float diag;                         // Film.diagonal, metres
    float area0;                        // exit_pupil_bounds[0].area()
    uint32_t n_el, simple;              // simple: "simpleweighting"
    float* weight;                      // k_raygen: the batch's per-slot camera ray weights (set at each launch), read by k_resolve<true>
};

// A ray through Transform::scale(1, 1, -1).transform_ray (realistic.rs:269,322): the matrix's entries as written, so that the
// products by 0 and their signs are those of the reference, and the origin pushed to the edge of its error bound (transform.rs:538-549).
PB_D void lens_flip_ray(V3& o, V3& d) {
    const float x = o.x, y = o.y, z = o.z;
    V3 op = mk3(1.0f * x + 0.0f * y + 0.0f * z + 0.0f, 0.0f * x + 1.0f * y + 0.0f * z + 0.0f, 0.0f * x + 0.0f * y + -1.0f * z + 0.0f);
    const float wp = 0.0f * x + 0.0f * y + 0.0f * z + 1.0f;
    const V3 err = mk3(fabsf(1.0f * x) + fabsf(0.0f * y) + fabsf(0.0f * z) + fabsf(0.0f), fabsf(0.0f * x) + fabsf(1.0f * y) + fabsf(0.0f * z) + fabsf(0.0f),
                       fabsf(0.0f * x) + fabsf(0.0f * y) + fabsf(-1.0f * z) + fabsf(0.0f)) * gamma_n(3);
    if (wp != 1.0f) op = vdiv(op, wp);
    const V3 dp = mk3(1.0f * d.x + 0.0f * d.y + 0.0f * d.z, 0.0f * d.x + 1.0f * d.y + 0.0f * d.z, 0.0f * d.x + 0.0f * d.y + -1.0f * d.z);
    const float ls = len2(dp);
    if (ls > 0.0f) op = op + dp * (dot3(abs3(dp), err) / ls);
    o = op;
    d = dp;
}

// RealisticCamera::trace_lenses_from_film (realistic.rs:266-327) with intersect_spherical_element (:328-365), quadratic's f64
// discriminant (pbrt.rs:248-268) and refract (reflection.rs:1897-1910).  o, d: a camera-space ray in, the camera-space ray out.
PB_D bool lens_trace_from_film(const DLens& L, V3& o, V3& d) {
    lens_flip_ray(o, d);
    float element_z = 0.0f;
    for (int i = (int)L.n_el - 1; i >= 0; --i) {
        const float4 e = L.el[i];
        element_z -= e.y;
        float t;
        V3 n = mk3(0.0f, 0.0f, 0.0f);
        const bool is_stop = e.x == 0.0f;
        if (is_stop) {
            if (d.z >= 0.0f) return false;
            t = (element_z - o.z) / d.z;
        } else {
            const float radius = e.x, z_center = element_z + e.x;
            const V3 oc = mk3(o.x - 0.0f, o.y - 0.0f, o.z - z_center);
            const float a = d.x * d.x + d.y * d.y + d.z * d.z;
            const float b = 2.0f * (d.x * oc.x + d.y * oc.y + d.z * oc.z);
            const float c = oc.x * oc.x + oc.y * oc.y + oc.z * oc.z - radius * radius;
            const double discrim = (double)b * (double)b - 4.0 * (double)a * (double)c;
            if (discrim < 0.0) return false;
            const double root = sqrt(discrim);
            const double q = b < 0.0f ? -0.5 * ((double)b - root) : -0.5 * ((double)b + root);
            float t0 = (float)q / a, t1 = c / (float)q;
            if (t0 > t1) { const float s = t0; t0 = t1; t1 = s; }
            const bool use_closer_t = (d.z > 0.0f) ^ (radius < 0.0f);
            t = use_closer_t ? fminf(t0, t1) : fmaxf(t0, t1);
            if (t < 0.0f) return false;
            n = faceforward3(norm3(oc + d * t), -d);
        }
        const V3 p_hit = o + d * t;
        const float r2 = p_hit.x * p_hit.x + p_hit.y * p_hit.y;
        if (r2 > e.w * e.w) return false;
        o = p_hit;
        if (!is_stop) {
            const float eta_i = e.z, eta_t = (i > 0 && L.el[i - 1].z != 0.0f) ? L.el[i - 1].z : 1.0f;
            const float eta = eta_i / eta_t;
            const V3 wi = norm3(-d);
            const float cos_i = n.x * wi.x + n.y * wi.y + n.z * wi.z;
            const float sin2_i = fmaxf(0.0f, 1.0f - cos_i * cos_i);
            const float sin2_t = eta * eta * sin2_i;
            if (sin2_t >= 1.0f) return false;
            const float cos_t = sqrtf(1.0f - sin2_t);
            d = (-wi) * eta + n * (eta * cos_i - cos_t);
        }
    }
    lens_flip_ray(o, d);
    return true;
}

// camera_to_world.transform_ray (transform.rs:538-549, origin error offset included) and the normalise of realistic.rs:234-235
PB_D void lens_to_world(const float* c, V3& o, V3& d) {
    const float x = o.x, y = o.y, z = o.z;
    V3 ow = mk3(c[0] * x + c[1] * y + c[2] * z + c[3], c[4] * x + c[5] * y + c[6] * z + c[7], c[8] * x + c[9] * y + c[10] * z + c[11]);
    const float wpc = c[12] * x + c[13] * y + c[14] * z + c[15];
    const V3 err = mk3(fabsf(c[0] * x) + fabsf(c[1] * y) + fabsf(c[2] * z) + fabsf(c[3]), fabsf(c[4] * x) + fabsf(c[5] * y) + fabsf(c[6] * z) + fabsf(c[7]),
                       fabsf(c[8] * x) + fabsf(c[9] * y) + fabsf(c[10] * z) + fabsf(c[11])) * gamma_n(3);
    if (wpc != 1.0f) ow = vdiv(ow, wpc);
    const V3 dw = mk3(c[0] * d.x + c[1] * d.y + c[2] * d.z, c[4] * d.x + c[5] * d.y + c[6] * d.z, c[8] * d.x + c[9] * d.y + c[10] * d.z);
    const float ls = len2(dw);
    if (ls > 0.0f) ow = ow + dw * (dot3(abs3(dw), err) / ls);
    o = ow;
    d = norm3(dw);
}

// RealisticCamera::generate_ray (realistic.rs:198-251): the world-space ray and its weight, 0 for a vignetted sample (o, d then
// unspecified).  c: camera_to_world at the sample's time; shutter: {open, close} for the non-simple weighting.
PB_D float lens_generate_ray(const DLens& L, const float* c, float2 shutter, float2 p_film, float2 p_lens, V3& o, V3& d) {
    const float sx = p_film.x / L.full_res.x, sy = p_film.y / L.full_res.y;
    const float fx = -lerpf(sx, L.ext_min.x, L.ext_max.x), fy = lerpf(sy, L.ext_min.y, L.ext_max.y);
    // sample_exit_pupil (:656-688)
    const float r_film = sqrtf(fx * fx + fy * fy);
    const float bin = floorf(r_film / (L.diag / 2.0f) * (float)PB_PUPIL_BINS);  // `as usize` saturates: NaN and negatives are 0
    const int r_index = bin >= (float)(PB_PUPIL_BINS - 1) ? PB_PUPIL_BINS - 1 : (bin > 0.0f ? (int)bin : 0);
    const float4 pb = L.pupil[r_index];
    const float area = (pb.z - pb.x) * (pb.w - pb.y);
    const float plx = lerpf(p_lens.x, pb.x, pb.z), ply = lerpf(p_lens.y, pb.y, pb.w);
    const float sin_t = r_film != 0.0f ? fy / r_film : 0.0f, cos_t = r_film != 0.0f ? fx / r_film : 1.0f;
    const float rear_z = L.el[L.n_el - 1].y;
    const V3 p_rear = mk3(cos_t * plx - sin_t * ply, sin_t * plx + cos_t * ply, rear_z);
    const V3 pf = mk3(fx, fy, 0.0f);
    const V3 d_film = p_rear - pf;
    o = pf;
    d = d_film;
    if (!lens_trace_from_film(L, o, d)) return 0.0f;
    lens_to_world(c, o, d);
    const float cos_theta = norm3(d_film).z;
    const float cos2 = cos_theta * cos_theta, cos4 = cos2 * cos2;
    if (L.simple) return cos4 * area / L.area0;
    return (shutter.y - shutter.x) * (cos4 * area) / (rear_z * rear_z);
}

// RealisticCamera::generate_ray_differential (realistic.rs:693-735): the main ray, then p_film shifted by +0.05 (-0.05 when that
// vignettes) in x and then in y.  The weight is 0 when the main ray or both shifts of one axis vignette; rxo..ryd are only
// written for a sample of weight > 0.  `rx_origin = o + (rx.o - o) / eps` divides by multiplying with 1 / eps (geometry.rs:1271).
PB_D float lens_generate_ray_differential(const DLens& L, const float* c, float2 shutter, float2 p_film, float2 p_lens, V3& o, V3& d, V3& rxo,
                                          V3& ryo, V3& rxd, V3& ryd) {
    const float wt = lens_generate_ray(L, c, shutter, p_film, p_lens, o, d);
    if (wt == 0.0f) return 0.0f;
    for (int axis = 0; axis < 2; ++axis) {
        float w = 0.0f;
        V3 so, sd;
        for (int k = 0; k < 2 && w == 0.0f; ++k) {
            const float eps = k == 0 ? 0.05f : -0.05f;
            const float2 ps = axis == 0 ? make_float2(p_film.x + eps, p_film.y) : make_float2(p_film.x, p_film.y + eps);
            w = lens_generate_ray(L, c, shutter, ps, p_lens, so, sd);
            if (w != 0.0f) {
                const float inv = 1.0f / eps;
                so = o + (so - o) * inv;
                sd = d + (sd - d) * inv;
            }
        }
        if (w == 0.0f) return 0.0f;
        if (axis == 0) { rxo = so; rxd = sd; }
        else { ryo = so; ryd = sd; }
    }
    return wt;
}

}  // namespace pb
