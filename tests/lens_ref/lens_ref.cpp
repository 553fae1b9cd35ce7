// TEST INFRASTRUCTURE ONLY.  The oracle (oracle/, included unchanged, through the cameras of tests/camera_ref and the animated camera
// of tests/motion_ref) extended by rs_pbrt's RealisticCamera::generate_ray_differential (src/cameras/realistic.rs:198-365,656-735),
// restated here from the reference independently of the library's pb_lens.cuh, and a per-sample render loop that runs li only for
// a camera ray weight > 0 and hands the weight to the film (integrator.rs:134-197).
// Built by tests/lens_ref.py into tests/lens_ref/_build/liblens_ref.so; nothing under rs_pbrt_b200/ uses it.
#include "../camera_ref/camera_ref.cpp"

namespace lref {

struct Lens {
    std::vector<PbrtLensElement> el;
    std::vector<float> pupil;  // 64 x {pmin.x, pmin.y, pmax.x, pmax.y}
    Float diagonal;
    bool simple;
    uint32_t full_res[2];
};

static const float kFlip[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, -1, 0, 0, 0, 0, 1};  // Transform::scale(1, 1, -1)

Float lerp_(Float t, Float a, Float b) { return a * (1.0f - t) + b * t; }  // pbrt.rs:235-245

// quadratic (pbrt.rs:248-268)
bool quadratic_lens(Float a, Float b, Float c, Float& t0, Float& t1) {
    const double discrim = (double)b * (double)b - 4.0 * (double)a * (double)c;
    if (discrim < 0.0) return false;
    const double root_discrim = std::sqrt(discrim);
    const double q = b < 0.0f ? -0.5 * ((double)b - root_discrim) : -0.5 * ((double)b + root_discrim);
    t0 = (Float)q / a;
    t1 = c / (Float)q;
    if (t0 > t1) std::swap(t0, t1);
    return true;
}

// intersect_spherical_element (:328-365)
bool intersect_spherical_element(Float radius, Float z_center, const Ray& ray, Float& t, Vec3& n) {
    const Point3 o = ray.o - Vec3(0.0f, 0.0f, z_center);
    const Float a = ray.d.x * ray.d.x + ray.d.y * ray.d.y + ray.d.z * ray.d.z;
    const Float b = 2.0f * (ray.d.x * o.x + ray.d.y * o.y + ray.d.z * o.z);
    const Float c = o.x * o.x + o.y * o.y + o.z * o.z - radius * radius;
    Float t0, t1;
    if (!quadratic_lens(a, b, c, t0, t1)) return false;
    const bool use_closer_t = (ray.d.z > 0.0f) ^ (radius < 0.0f);
    t = use_closer_t ? std::fmin(t0, t1) : std::fmax(t0, t1);
    if (t < 0.0f) return false;
    n = normalize(o + ray.d * t);
    const Vec3 v = -ray.d;
    if (n.x * v.x + n.y * v.y + n.z * v.z < 0.0f) n = -n;  // nrm_faceforward_vec3
    return true;
}

// refract (reflection.rs:1897-1910)
bool refract_lens(const Vec3& wi, const Vec3& n, Float eta, Vec3& wt) {
    const Float cos_theta_i = n.x * wi.x + n.y * wi.y + n.z * wi.z;
    const Float sin2_theta_i = std::fmax(0.0f, 1.0f - cos_theta_i * cos_theta_i);
    const Float sin2_theta_t = eta * eta * sin2_theta_i;
    if (sin2_theta_t >= 1.0f) return false;
    const Float cos_theta_t = std::sqrt(1.0f - sin2_theta_t);
    wt = -wi * eta + n * (eta * cos_theta_i - cos_theta_t);
    return true;
}

// trace_lenses_from_film (:266-327)
bool trace_lenses_from_film(const Lens& L, const Ray& r_camera, Ray* r_out) {
    Float element_z = 0.0f;
    Ray r_lens = xf_ray(kFlip, r_camera);
    const size_t n = L.el.size();
    for (size_t idx = 0; idx < n; ++idx) {
        const size_t i = n - 1 - idx;
        const PbrtLensElement& element = L.el[i];
        element_z -= element.thickness;
        Float t = 0.0f;
        Vec3 nrm;
        const bool is_stop = element.curvature_radius == 0.0f;
        if (is_stop) {
            if (r_lens.d.z >= 0.0f) return false;
            t = (element_z - r_lens.o.z) / r_lens.d.z;
        } else if (!intersect_spherical_element(element.curvature_radius, element_z + element.curvature_radius, r_lens, t, nrm)) return false;
        const Point3 p_hit = r_lens.o + r_lens.d * t;
        if (p_hit.x * p_hit.x + p_hit.y * p_hit.y > element.aperture_radius * element.aperture_radius) return false;
        r_lens.o = p_hit;
        if (!is_stop) {
            const Float eta_i = element.eta;
            const Float eta_t = (i > 0 && L.el[i - 1].eta != 0.0f) ? L.el[i - 1].eta : 1.0f;
            Vec3 w;
            if (!refract_lens(normalize(-r_lens.d), nrm, eta_i / eta_t, w)) return false;
            r_lens.d = w;
        }
    }
    if (r_out) *r_out = xf_ray(kFlip, r_lens);
    return true;
}

// generate_ray (:198-251) with sample_exit_pupil (:656-688) and Film::get_physical_extent (film.rs:293-307).  c2w: camera_to_world
// at the sample's time.
Float generate_ray(const Lens& L, const float* c2w, Float shutter_open, Float shutter_close, const Vec2& sp_film, const Vec2& p_lens, Float time, Ray& ray) {
    const Vec2 s(sp_film.x / (Float)L.full_res[0], sp_film.y / (Float)L.full_res[1]);
    const Float aspect = (Float)L.full_res[1] / (Float)L.full_res[0];
    const Float ex = std::sqrt(L.diagonal * L.diagonal / (1.0f + aspect * aspect)), ey = aspect * ex;
    const Vec2 p_film2(lerp_(s.x, -ex / 2.0f, ex / 2.0f), lerp_(s.y, -ey / 2.0f, ey / 2.0f));
    const Point3 p_film(-p_film2.x, p_film2.y, 0.0f);
    // sample_exit_pupil
    const Float r_film = std::sqrt(p_film.x * p_film.x + p_film.y * p_film.y);
    const Float fi = std::floor(r_film / (L.diagonal / 2.0f) * 64.0f);
    size_t r_index = fi != fi || fi <= 0.0f ? 0 : (fi >= 1.8e19f ? SIZE_MAX : (size_t)fi);  // Rust's saturating `as usize`
    r_index = std::min<size_t>(63, r_index);
    const float* pb = L.pupil.data() + 4 * r_index;
    const Float area = (pb[2] - pb[0]) * (pb[3] - pb[1]);
    const Vec2 pl(lerp_(p_lens.x, pb[0], pb[2]), lerp_(p_lens.y, pb[1], pb[3]));
    const Float sin_theta = r_film != 0.0f ? p_film.y / r_film : 0.0f;
    const Float cos_theta = r_film != 0.0f ? p_film.x / r_film : 1.0f;
    const Point3 p_rear(cos_theta * pl.x - sin_theta * pl.y, sin_theta * pl.x + cos_theta * pl.y, L.el.back().thickness);
    const Ray r_film_ray(p_film, p_rear - p_film, INF, lerp_(time, shutter_open, shutter_close));
    Ray out;
    if (!trace_lenses_from_film(L, r_film_ray, &out)) return 0.0f;
    out.time = r_film_ray.time;
    ray = xf_ray(c2w, out);
    ray.d = normalize(ray.d);
    const Float ct = normalize(r_film_ray.d).z;
    const Float c2 = ct * ct, c4 = c2 * c2;
    if (L.simple) {
        const Float area0 = (L.pupil[2] - L.pupil[0]) * (L.pupil[3] - L.pupil[1]);
        return c4 * area / area0;
    }
    const Float rz = L.el.back().thickness;
    return (shutter_close - shutter_open) * (c4 * area) / (rz * rz);
}

// generate_ray_differential (:693-735)
Float generate_ray_differential(const Lens& L, const float* c2w, Float so, Float sc, const Vec2& p_film, const Vec2& p_lens, Float time, Ray& ray) {
    const Float wt = generate_ray(L, c2w, so, sc, p_film, p_lens, time, ray);
    if (wt == 0.0f) return 0.0f;
    const Float eps_values[2] = {0.05f, -0.05f};
    Float wtx = 0.0f;
    for (Float eps : eps_values) {
        Ray rx;
        wtx = generate_ray(L, c2w, so, sc, Vec2(p_film.x + eps, p_film.y), p_lens, time, rx);
        ray.rx_origin = ray.o + (rx.o - ray.o) / eps;
        ray.rx_direction = ray.d + (rx.d - ray.d) / eps;
        if (wtx != 0.0f) break;
    }
    if (wtx == 0.0f) return 0.0f;
    Float wty = 0.0f;
    for (Float eps : eps_values) {
        Ray ry;
        wty = generate_ray(L, c2w, so, sc, Vec2(p_film.x, p_film.y + eps), p_lens, time, ry);
        ray.ry_origin = ray.o + (ry.o - ray.o) / eps;
        ray.ry_direction = ray.d + (ry.d - ray.d) / eps;
        if (wty != 0.0f) break;
    }
    if (wty == 0.0f) return 0.0f;
    ray.has_differential = true;
    return wt;
}

Lens make_lens(const PbrtRealisticLens* lens, const uint32_t full_res[2]) {
    Lens L;
    L.el.assign(lens->elements, lens->elements + lens->n_elements);
    L.pupil.assign(lens->exit_pupil_bounds, lens->exit_pupil_bounds + 256);
    L.diagonal = lens->film_diagonal;
    L.simple = lens->simple_weighting != 0;
    L.full_res[0] = full_res[0]; L.full_res[1] = full_res[1];
    return L;
}

}  // namespace lref

extern "C" {

// generate_ray_differential of n camera samples through camera_to_world (animated when cam_motion != NULL), before the 1/sqrt(spp)
// scale: 19 floats per sample, o[3] d[3] weight rx_o[3] ry_o[3] rx_d[3] ry_d[3], zeros where the weight is 0.
int lref_camera_rays(const PbrtCamera* cam, const PbrtRealisticLens* lens, const uint32_t full_res[2], const PbrtAnimatedTransform* cam_motion, uint32_t n,
                     const float* p_film, const float* p_lens, const float* time, float* out) {
    const lref::Lens L = lref::make_lens(lens, full_res);
    std::unique_ptr<mref::Animated> at(cam_motion ? new mref::Animated(*cam_motion) : nullptr);
    for (uint32_t i = 0; i < n; ++i) {
        float c2w[16];
        std::memcpy(c2w, cam->camera_to_world, 64);
        if (at) {
            mref::Mat m, mi;
            at->interpolate(lerp(time[i], cam->shutter_open, cam->shutter_close), m, mi);
            std::memcpy(c2w, m, 64);
        }
        Ray r;
        const Float w = lref::generate_ray_differential(L, c2w, cam->shutter_open, cam->shutter_close, Vec2(p_film[2 * i], p_film[2 * i + 1]),
                                                        Vec2(p_lens[2 * i], p_lens[2 * i + 1]), time[i], r);
        float v[19] = {0};
        if (w != 0.0f) {
            const float a[19] = {r.o.x, r.o.y, r.o.z, r.d.x, r.d.y, r.d.z, w, r.rx_origin.x, r.rx_origin.y, r.rx_origin.z, r.ry_origin.x, r.ry_origin.y,
                                 r.ry_origin.z, r.rx_direction.x, r.rx_direction.y, r.rx_direction.z, r.ry_direction.x, r.ry_direction.y, r.ry_direction.z};
            std::memcpy(v, a, sizeof v);
        } else v[6] = w;
        std::memcpy(out + 19 * (size_t)i, v, sizeof v);
    }
    return 0;
}

// cref_render's loop for the realistic camera: li only for a weight > 0, L * weight * filter weight into the film (integrator.rs:157-186).
// sample_rgb / sample_weight (optional): li's L (0 for a vignetted sample) and the camera ray weight, [pixel in rect][sample].
int lref_render(void* scene, const PbrtRealisticLens* lens, const uint32_t full_res[2], const PbrtAnimatedTransform* cam_motion, const PbrtRenderParams* rpp,
                const int32_t rect[4], float* film_rgbw, float* sample_rgb, float* sample_weight, PbrtStats* stats) {
    if (!sobol_tables().loaded) return fail("orc_init not called");
    try {
        const Scene& sc = *(Scene*)scene;
        const PbrtRenderParams& rp = *rpp;
        const lref::Lens Ln = lref::make_lens(lens, full_res);
        std::unique_ptr<mref::Animated> at(cam_motion ? new mref::Animated(*cam_motion) : nullptr);
        sc.instancing = rp.instancing;
        LightDistribution ld(&sc, (int)rp.light_strategy);
        const bool is_direct = rp.integrator == PBRT_INTEGRATOR_DIRECT || rp.integrator == PBRT_INTEGRATOR_WHITTED;
        DirectCfg dcfg;
        dcfg.whitted = rp.integrator == PBRT_INTEGRATOR_WHITTED;
        dcfg.sample_all = rp.direct_strategy == PBRT_DIRECT_SAMPLE_ALL;
        dcfg.max_depth = rp.max_depth;
        for (const AreaLight& l : sc.lights) dcfg.n_light_samples.push_back((int32_t)std::max(1u, l.n_samples));
        sc.allow_multiple_lobes = !is_direct;
        Counters cnt;
        std::unique_ptr<Sampler> sampler_owner = make_sampler(rp);
        Sampler& sampler = *sampler_owner;
        if (rp.integrator == PBRT_INTEGRATOR_AO) sampler.request_2d_array((int32_t)rp.ao_samples);
        if (is_direct && dcfg.sample_all && !dcfg.whitted)
            for (uint32_t i = 0; i < dcfg.max_depth; ++i)
                for (size_t j = 0; j < sc.lights.size(); ++j) {
                    sampler.request_2d_array(dcfg.n_light_samples[j]);
                    sampler.request_2d_array(dcfg.n_light_samples[j]);
                }
        ShadeCtx cx{&sc, &sampler, &ld, &cnt};
        const int32_t rw = rect[2] - rect[0];
        for (int32_t py = rect[1]; py < rect[3]; ++py)
            for (int32_t px = rect[0]; px < rect[2]; ++px) {
                sampler.start_pixel(px, py);
                if (!(px >= rp.pixel_bounds[0] && px < rp.pixel_bounds[2] && py >= rp.pixel_bounds[1] && py < rp.pixel_bounds[3])) continue;
                bool more = true;
                while (more) {
                    const int64_t si = sampler.current_pixel_sample_index;
                    Vec2 u = sampler.get_2d();
                    Vec2 p_film((Float)px + u.x, (Float)py + u.y);
                    Float time = sampler.get_1d();
                    Vec2 p_lens = sampler.get_2d();
                    const PbrtCamera& c = sc.camera;
                    float c2w[16];
                    std::memcpy(c2w, c.camera_to_world, 64);
                    if (at) {
                        mref::Mat m, mi;
                        at->interpolate(lerp(time, c.shutter_open, c.shutter_close), m, mi);
                        std::memcpy(c2w, m, 64);
                    }
                    Ray ray;
                    const Float w = lref::generate_ray_differential(Ln, c2w, c.shutter_open, c.shutter_close, p_film, p_lens, time, ray);
                    ray.scale_differentials(1.0f / std::sqrt((Float)rp.spp));
                    Spectrum l(0.0f);
                    if (w > 0.0f) {
                        cnt.camera_rays++;
                        l = rp.integrator == PBRT_INTEGRATOR_AO ? ao_li(cx, ray, (int32_t)rp.ao_samples, rp.ao_cos_sample != 0)
                            : is_direct                        ? direct_li(cx, dcfg, ray, 0)
                                                               : path_li(cx, ray, rp.max_depth, rp.rr_threshold);
                    }
                    if (l.has_nans()) l = Spectrum(0.0f);
                    const size_t k = ((size_t)(py - rect[1]) * (size_t)rw + (size_t)(px - rect[0])) * rp.spp + (size_t)si;
                    if (sample_rgb) { sample_rgb[3 * k] = l.c[0]; sample_rgb[3 * k + 1] = l.c[1]; sample_rgb[3 * k + 2] = l.c[2]; }
                    if (sample_weight) sample_weight[k] = w;
                    if (film_rgbw) film_add_sample(rp, film_rgbw, p_film, l, w);
                    more = sampler.start_next_sample();
                }
            }
        fill_stats(stats, cnt);
    } catch (const std::exception& e) { return fail(e.what()); }
    return 0;
}

}  // extern "C"
