// TEST INFRASTRUCTURE ONLY.  The oracle (oracle/, included unchanged) extended by an animated camera: AnimatedTransform restated
// from rs_pbrt (src/core/transform.rs:893-940, 2032-2124; src/core/quaternion.rs) independently of the library's pb_motion.cuh, and a
// per-sample render loop whose camera rays go through camera_to_world interpolated at each sample's time.  Built by
// tests/motion_ref.py into tests/motion_ref/_build/libmotion_ref.so; nothing under rs_pbrt_b200/ uses it.
#include "../../oracle/oracle_api.cpp"

#include <cmath>

namespace mref {

typedef float Mat[4][4];

void matmul(const Mat a, const Mat b, Mat out) {  // mtx_mul, transform.rs:238-249
    Mat r;
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) r[i][j] = a[i][0] * b[0][j] + a[i][1] * b[1][j] + a[i][2] * b[2][j] + a[i][3] * b[3][j];
    std::memcpy(out, r, sizeof r);
}

void invert(const Mat m, Mat out) {  // Matrix4x4::inverse, transform.rs:128-201
    int indxc[4], indxr[4], ipiv[4] = {0, 0, 0, 0};
    Mat minv;
    std::memcpy(minv, m, sizeof minv);
    for (int i = 0; i < 4; ++i) {
        int irow = 0, icol = 0;
        float big = 0.0f;
        for (int j = 0; j < 4; ++j) {
            if (ipiv[j] == 1) continue;
            for (int k = 0; k < 4; ++k)
                if (ipiv[k] == 0 && std::fabs(minv[j][k]) >= big) { big = std::fabs(minv[j][k]); irow = j; icol = k; }
        }
        ipiv[icol] += 1;
        if (irow != icol) std::swap(minv[irow], minv[icol]);
        indxr[i] = irow;
        indxc[i] = icol;
        float pivinv = 1.0f / minv[icol][icol];
        minv[icol][icol] = 1.0f;
        for (int j = 0; j < 4; ++j) minv[icol][j] *= pivinv;
        for (int j = 0; j < 4; ++j) {
            if (j == icol) continue;
            float save = minv[j][icol];
            minv[j][icol] = 0.0f;
            for (int k = 0; k < 4; ++k) minv[j][k] -= minv[icol][k] * save;
        }
    }
    for (int j = 3; j >= 0; --j)
        if (indxr[j] != indxc[j])
            for (int k = 0; k < 4; ++k) std::swap(minv[k][indxr[j]], minv[k][indxc[j]]);
    std::memcpy(out, minv, sizeof minv);
}

struct Quat { float v[3]; float w; };
float qdot(const Quat& a, const Quat& b) { return a.v[0] * b.v[0] + a.v[1] * b.v[1] + a.v[2] * b.v[2] + a.w * b.w; }
Quat qnormalize(const Quat& q) {  // Quaternion / f32: Vector3f's `/` multiplies by the reciprocal (geometry.rs:1271-1279)
    float len = std::sqrt(qdot(q, q));
    float inv = 1.0f / len;
    return Quat{{q.v[0] * inv, q.v[1] * inv, q.v[2] * inv}, q.w / len};
}
Quat qcombine(const Quat& a, float sa, const Quat& b, float sb) {
    return Quat{{a.v[0] * sa + b.v[0] * sb, a.v[1] * sa + b.v[1] * sb, a.v[2] * sa + b.v[2] * sb}, a.w * sa + b.w * sb};
}

Quat quat_from(const Mat m) {  // Quaternion::new, quaternion.rs:34-79
    float trace = m[0][0] + m[1][1] + m[2][2];
    if (trace > 0.0f) {
        float s = std::sqrt(trace + 1.0f);
        float w = s / 2.0f;
        s = 0.5f / s;
        return Quat{{(m[2][1] - m[1][2]) * s, (m[0][2] - m[2][0]) * s, (m[1][0] - m[0][1]) * s}, w};
    }
    static const int nxt[3] = {1, 2, 0};
    float q[3] = {0, 0, 0};
    int i = m[1][1] > m[0][0] ? 1 : 0;
    if (m[2][2] > m[i][i]) i = 2;
    int j = nxt[i], k = nxt[j];
    float s = std::sqrt((m[i][i] - (m[j][j] + m[k][k])) + 1.0f);
    q[i] = s * 0.5f;
    if (s != 0.0f) s = 0.5f / s;
    float w = (m[k][j] - m[j][k]) * s;
    q[j] = (m[j][i] + m[i][j]) * s;
    q[k] = (m[k][i] + m[i][k]) * s;
    return Quat{{q[0], q[1], q[2]}, w};
}

void decompose(const Mat m, float t[3], Quat& rq, Mat s) {  // AnimatedTransform::decompose, transform.rs:2032-2080
    t[0] = m[0][3]; t[1] = m[1][3]; t[2] = m[2][3];
    Mat r;
    std::memcpy(r, m, sizeof r);
    for (int i = 0; i < 3; ++i) r[i][3] = r[3][i] = 0.0f;
    r[3][3] = 1.0f;
    int count = 0;
    float norm;
    do {
        Mat rt, rit, rnext;
        for (int i = 0; i < 4; ++i)
            for (int j = 0; j < 4; ++j) rt[i][j] = r[j][i];
        invert(rt, rit);
        for (int i = 0; i < 4; ++i)
            for (int j = 0; j < 4; ++j) rnext[i][j] = 0.5f * (r[i][j] + rit[i][j]);
        norm = 0.0f;
        for (int i = 0; i < 3; ++i) {
            float n = std::fabs(r[i][0] - rnext[i][0]) + std::fabs(r[i][1] - rnext[i][1]) + std::fabs(r[i][2] - rnext[i][2]);
            norm = std::fmax(norm, n);
        }
        std::memcpy(r, rnext, sizeof r);
        ++count;
    } while (count < 100 && norm > 0.0001f);
    rq = quat_from(r);
    Mat rinv;
    invert(r, rinv);
    matmul(rinv, m, s);
}

struct Animated {
    Mat m0, m0_inv, m1, m1_inv;
    float t0, t1;
    bool animated;
    float tr[2][3];
    Quat rot[2];
    Mat sc[2];
    explicit Animated(const PbrtAnimatedTransform& a) {  // AnimatedTransform::new, transform.rs:912-932
        std::memcpy(m0, a.start, 64); std::memcpy(m0_inv, a.start_inv, 64);
        std::memcpy(m1, a.end, 64); std::memcpy(m1_inv, a.end_inv, 64);
        t0 = a.start_time; t1 = a.end_time;
        animated = false;
        for (int k = 0; k < 16; ++k) animated = animated || a.start[k] != a.end[k] || a.start_inv[k] != a.end_inv[k];
        decompose(m0, tr[0], rot[0], sc[0]);
        decompose(m1, tr[1], rot[1], sc[1]);
        if (qdot(rot[0], rot[1]) < 0.0f) rot[1] = Quat{{-rot[1].v[0], -rot[1].v[1], -rot[1].v[2]}, -rot[1].w};
    }
    void interpolate(float time, Mat m, Mat m_inv) const {  // AnimatedTransform::interpolate, transform.rs:2081-2113
        if (!animated || time <= t0) { std::memcpy(m, m0, 64); std::memcpy(m_inv, m0_inv, 64); return; }
        if (time >= t1) { std::memcpy(m, m1, 64); std::memcpy(m_inv, m1_inv, 64); return; }
        float dt = (time - t0) / (t1 - t0);
        float trans[3];
        for (int k = 0; k < 3; ++k) trans[k] = tr[0][k] * (1.0f - dt) + tr[1][k] * dt;
        // quat_slerp, quaternion.rs:168-178
        Quat q;
        float cos_theta = qdot(rot[0], rot[1]);
        if (cos_theta > 0.9995f) {
            q = qnormalize(qcombine(rot[0], 1.0f - dt, rot[1], dt));
        } else {
            float theta = std::acos(orc::clamp_t(cos_theta, -1.0f, 1.0f));
            float thetap = theta * dt;
            Quat qperp = qnormalize(qcombine(rot[1], 1.0f, rot[0], -cos_theta));
            q = qcombine(rot[0], std::cos(thetap), qperp, std::sin(thetap));
        }
        Mat scale = {{0, 0, 0, 0}, {0, 0, 0, 0}, {0, 0, 0, 0}, {0, 0, 0, 1}}, scale_inv;
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) scale[i][j] = orc::lerp(dt, sc[0][i][j], sc[1][i][j]);
        invert(scale, scale_inv);
        // Quaternion::to_transform, quaternion.rs:80-107
        const float x = q.v[0], y = q.v[1], z = q.v[2], w = q.w;
        Mat a = {{1.0f - 2.0f * (y * y + z * z), 2.0f * (x * y + z * w), 2.0f * (x * z - y * w), 0.0f},
                 {2.0f * (x * y - z * w), 1.0f - 2.0f * (x * x + z * z), 2.0f * (y * z + x * w), 0.0f},
                 {2.0f * (x * z + y * w), 2.0f * (y * z - x * w), 1.0f - 2.0f * (x * x + y * y), 0.0f},
                 {0.0f, 0.0f, 0.0f, 1.0f}};
        Mat at;
        for (int i = 0; i < 4; ++i)
            for (int j = 0; j < 4; ++j) at[i][j] = a[j][i];
        Mat tm = {{1, 0, 0, trans[0]}, {0, 1, 0, trans[1]}, {0, 0, 1, trans[2]}, {0, 0, 0, 1}};
        Mat tm_inv = {{1, 0, 0, -trans[0]}, {0, 1, 0, -trans[1]}, {0, 0, 1, -trans[2]}, {0, 0, 0, 1}};
        Mat p, p_inv;
        matmul(tm, at, p);          // Transform::translate(trans) * rotate.to_transform()
        matmul(a, tm_inv, p_inv);
        matmul(p, scale, m);        // ... * Transform {scale, inverse(scale)}
        matmul(scale_inv, p_inv, m_inv);
    }
};

}  // namespace mref

extern "C" {

// AnimatedTransform::new + interpolate at n times: 16 floats of m and of m_inv per time
int mref_interpolate(const PbrtAnimatedTransform* a, uint32_t n, const float* times, float* m_out, float* m_inv_out) {
    mref::Animated at(*a);
    for (uint32_t i = 0; i < n; ++i) {
        mref::Mat m, mi;
        at.interpolate(times[i], m, mi);
        std::memcpy(m_out + 16 * (size_t)i, m, 64);
        std::memcpy(m_inv_out + 16 * (size_t)i, mi, 64);
    }
    return 0;
}

// decompose(m): t[3], q = {x, y, z, w}, s[16]
void mref_decompose(const float* m16, float* t3, float* q4, float* s16) {
    mref::Mat m, s;
    std::memcpy(m, m16, 64);
    mref::Quat q;
    mref::decompose(m, t3, q, s);
    q4[0] = q.v[0]; q4[1] = q.v[1]; q4[2] = q.v[2]; q4[3] = q.w;
    std::memcpy(s16, s, 64);
}

// orc_render for a scene seen by an animated camera (cam == NULL: static): SamplerIntegrator::render's per-sample work
// (integrator.rs:123-197) with PerspectiveCamera::generate_ray_differential's final camera_to_world.transform_ray going through
// the camera's AnimatedTransform at ray.time.  Single-threaded, pixels of `rect` in row-major order, so that the film's sums run in
// sample order.  sample_rgb / sample_time (optional): radiance and ray.time of every sample, [pixel in rect][sample].
int mref_render(void* scene, const PbrtAnimatedTransform* cam, const PbrtRenderParams* rpp, const int32_t rect[4], float* film_rgbw,
                float* sample_rgb, float* sample_time, PbrtStats* stats) {
    if (!sobol_tables().loaded) return fail("orc_init not called");
    try {
        const Scene& sc = *(Scene*)scene;
        const PbrtRenderParams& rp = *rpp;
        std::unique_ptr<mref::Animated> at(cam ? new mref::Animated(*cam) : nullptr);
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
                    PbrtCamera c = sc.camera;
                    const Float ray_time = lerp(time, c.shutter_open, c.shutter_close);  // perspective.rs:226
                    if (at) {
                        mref::Mat m, mi;
                        at->interpolate(ray_time, m, mi);
                        std::memcpy(c.camera_to_world, m, 64);
                    }
                    Ray ray = camera_ray(c, p_film, time, p_lens);
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
