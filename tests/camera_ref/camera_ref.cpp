// TEST INFRASTRUCTURE ONLY.  The oracle (oracle/, included unchanged, through the animated camera of tests/motion_ref) extended by
// rs_pbrt's OrthographicCamera (src/cameras/orthographic.rs:38-235) and EnvironmentCamera (src/cameras/environment.rs:92-116),
// restated here from the reference independently of the library's k_raygen, and a per-sample render loop that traces their rays.
// Built by tests/camera_ref.py into tests/camera_ref/_build/libcamera_ref.so; nothing under rs_pbrt_b200/ uses it.
#include "../motion_ref/motion_ref.cpp"

namespace cref {

// OrthographicCamera::generate_ray_differential, orthographic.rs:156-230.  dx_camera / dy_camera are raster_to_camera.transform_vector
// of the unit raster steps (OrthographicCamera::new, :75-84).
Ray orthographic_ray(const PbrtCamera& cam, const Vec2& p_film, Float time, const Vec2& p_lens) {
    const Vec3 dx_camera = xf_vector(cam.raster_to_camera, Vec3(1.0f, 0.0f, 0.0f));
    const Vec3 dy_camera = xf_vector(cam.raster_to_camera, Vec3(0.0f, 1.0f, 0.0f));
    const Point3 p_camera = xf_point(cam.raster_to_camera, Point3(p_film.x, p_film.y, 0.0f));
    Ray ray(p_camera, Vec3(0.0f, 0.0f, 1.0f), INF, lerp(time, cam.shutter_open, cam.shutter_close));
    if (cam.lens_radius > 0.0f) {  // :177-188
        Vec2 pl = concentric_sample_disk(p_lens);
        pl = Vec2(pl.x * cam.lens_radius, pl.y * cam.lens_radius);
        const Float ft = cam.focal_distance / ray.d.z;
        const Point3 p_focus = ray.o + ray.d * ft;  // Ray::position
        ray.o = Point3(pl.x, pl.y, 0.0f);
        ray.d = normalize(p_focus - ray.o);
    }
    ray.has_differential = true;
    if (cam.lens_radius > 0.0f) {  // :190-211, as written: ft from the updated ray.d, one p_focus (dx_camera's) for rx and ry
        Vec2 pl = concentric_sample_disk(p_lens);
        pl = Vec2(pl.x * cam.lens_radius, pl.y * cam.lens_radius);
        const Float ft = cam.focal_distance / ray.d.z;
        const Point3 p_focus = p_camera + dx_camera + Vec3(0.0f, 0.0f, 1.0f) * ft;
        ray.rx_origin = Point3(pl.x, pl.y, 0.0f);
        ray.ry_origin = Point3(pl.x, pl.y, 0.0f);
        ray.rx_direction = normalize(p_focus - ray.rx_origin);
        ray.ry_direction = normalize(p_focus - ray.ry_origin);
    } else {  // :212-220
        ray.rx_origin = ray.o + dx_camera;
        ray.ry_origin = ray.o + dy_camera;
        ray.rx_direction = ray.d;
        ray.ry_direction = ray.d;
    }
    return xf_ray(cam.camera_to_world, ray);
}

// EnvironmentCamera::generate_ray_differential, environment.rs:92-116: no differential
Ray environment_ray(const PbrtCamera& cam, const uint32_t full_res[2], const Vec2& p_film, Float time) {
    const Float theta = PI * p_film.y / (Float)full_res[1];
    const Float phi = 2.0f * PI * p_film.x / (Float)full_res[0];
    const Vec3 dir(std::sin(theta) * std::cos(phi), std::cos(theta), std::sin(theta) * std::sin(phi));
    const Ray in_ray(Point3(0.0f, 0.0f, 0.0f), dir, INF, lerp(time, cam.shutter_open, cam.shutter_close));
    return xf_ray(cam.camera_to_world, in_ray);
}

Ray generate(const PbrtCamera& cam, uint32_t kind, const uint32_t full_res[2], const Vec2& p_film, Float time, const Vec2& p_lens) {
    if (kind == PBRT_CAMERA_ORTHOGRAPHIC) return orthographic_ray(cam, p_film, time, p_lens);
    if (kind == PBRT_CAMERA_ENVIRONMENT) return environment_ray(cam, full_res, p_film, time);
    return camera_ray(cam, p_film, time, p_lens);  // the oracle's PerspectiveCamera
}

}  // namespace cref

extern "C" {

// The camera ray of each (p_film, time, p_lens) as the integrator hands it on: after camera_to_world and the 1/sqrt(spp) differential
// scale (integrator.rs:140-144).  Per ray: o[3], d[3], time, has_diff, rx_o[3], ry_o[3], rx_d[3], ry_d[3] = 20 floats.
int cref_camera_rays(const PbrtCamera* cam, uint32_t kind, const uint32_t full_res[2], uint32_t spp, uint32_t n, const float* p_film, const float* time,
                     const float* p_lens, float* out) {
    for (uint32_t i = 0; i < n; ++i) {
        Ray r = cref::generate(*cam, kind, full_res, Vec2(p_film[2 * i], p_film[2 * i + 1]), time[i], Vec2(p_lens[2 * i], p_lens[2 * i + 1]));
        r.scale_differentials(1.0f / std::sqrt((Float)spp));
        const float v[20] = {r.o.x, r.o.y, r.o.z, r.d.x, r.d.y, r.d.z, r.time, r.has_differential ? 1.0f : 0.0f,
                             r.rx_origin.x, r.rx_origin.y, r.rx_origin.z, r.ry_origin.x, r.ry_origin.y, r.ry_origin.z,
                             r.rx_direction.x, r.rx_direction.y, r.rx_direction.z, r.ry_direction.x, r.ry_direction.y, r.ry_direction.z};
        std::memcpy(out + 20 * (size_t)i, v, sizeof v);
    }
    return 0;
}

// orc_render for a scene seen by camera `kind` (PbrtCameraKind; full_res = Film.full_resolution), animated when cam_motion != NULL:
// the per-sample loop of mref_render with the camera's own generate_ray_differential.  Single-threaded, pixels of `rect` in row-major
// order.  sample_rgb / sample_time (optional): radiance and ray.time of every sample, [pixel in rect][sample].
int cref_render(void* scene, uint32_t kind, const uint32_t full_res[2], const PbrtAnimatedTransform* cam_motion, const PbrtRenderParams* rpp,
                const int32_t rect[4], float* film_rgbw, float* sample_rgb, float* sample_time, PbrtStats* stats) {
    if (!sobol_tables().loaded) return fail("orc_init not called");
    try {
        const Scene& sc = *(Scene*)scene;
        const PbrtRenderParams& rp = *rpp;
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
                    Vec2 u = sampler.get_2d();  // CameraSample (sampler.rs:85-95)
                    Vec2 p_film((Float)px + u.x, (Float)py + u.y);
                    Float time = sampler.get_1d();
                    Vec2 p_lens = sampler.get_2d();
                    PbrtCamera c = sc.camera;
                    if (at) {  // camera_to_world.transform_ray is the AnimatedTransform's, at ray.time
                        mref::Mat m, mi;
                        at->interpolate(lerp(time, c.shutter_open, c.shutter_close), m, mi);
                        std::memcpy(c.camera_to_world, m, 64);
                    }
                    Ray ray = cref::generate(c, kind, full_res, p_film, time, p_lens);
                    ray.scale_differentials(1.0f / std::sqrt((Float)rp.spp));
                    cnt.camera_rays++;
                    Spectrum l = rp.integrator == PBRT_INTEGRATOR_AO ? ao_li(cx, ray, (int32_t)rp.ao_samples, rp.ao_cos_sample != 0)
                                 : is_direct                        ? direct_li(cx, dcfg, ray, 0)
                                                                    : path_li(cx, ray, rp.max_depth, rp.rr_threshold);
                    if (l.has_nans()) l = Spectrum(0.0f);
                    const size_t k = ((size_t)(py - rect[1]) * (size_t)rw + (size_t)(px - rect[0])) * rp.spp + (size_t)si;
                    if (sample_rgb) { sample_rgb[3 * k] = l.c[0]; sample_rgb[3 * k + 1] = l.c[1]; sample_rgb[3 * k + 2] = l.c[2]; }
                    if (sample_time) sample_time[k] = ray.time;
                    if (film_rgbw) film_add_sample(rp, film_rgbw, p_film, l, 1.0f);
                    more = sampler.start_next_sample();
                }
            }
        fill_stats(stats, cnt);
    } catch (const std::exception& e) { return fail(e.what()); }
    return 0;
}

}  // extern "C"
