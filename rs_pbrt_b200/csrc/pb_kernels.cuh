// pb_kernels.cuh -- the wavefront kernels of the PathIntegrator hot path (sm_90a).
//
// One batch = up to `capacity` camera samples (whole pixels x all their spp).  Per batch:
//   k_raygen                       SobolSampler::start_pixel/get_camera_sample + PerspectiveCamera ray -> ray queue
//   repeat (max_depth + 1 times, or until the queues drain when null materials exist):
//     k_trace  (dominant kernel)   persistent ray caster over the unified ray queue (path, MIS and shadow
//                                  rays; one ray per lane, while-while traversal, per-lane refill)
//     k_voxel_request / k_lightgrid_contrib / k_lightgrid_build
//                                  SpatialLightDistribution::compute_distribution for first-touched voxels
//     k_shade                      resolves the previous vertex's next-event estimate (shadow + MIS results),
//                                  then one vertex of PathIntegrator::li: Le, uniform_sample_one_light /
//                                  estimate_direct set-up, Bsdf::sample_f, Russian roulette; emits up to three
//                                  rays and compacts survivors (warp ballot + prefix sum)
//   k_resolve                      FilmTile::add_sample in sample order, one thread per pixel
#pragma once
#include "pb_bsdf.cuh"
#include "pb_interaction.cuh"
#include "pb_sobol.cuh"
#include "pb_texture.cuh"
#include "pb_material.cuh"
#include "pb_motion.cuh"
#include "pb_lens.cuh"

namespace pb {

#define PB_TRACE_THREADS 128
#define PB_TRACE_SMEM_BYTES 49152  // scenes whose nodes + triangles fit are traced entirely out of shared memory
#define PB_SHADE_THREADS 128
#define PB_SMEM_SOBOL_BYTES 49152  // budget for the Sobol' nibble-table slice staged in shared memory by TMA

// ---- TMA 1-D bulk copy global -> shared, completion on an mbarrier ---------------------------
#ifdef PB_HOST_EMU
// tests/emu (kernel-logic emulation on the CPU, test infrastructure): the copying thread copies, the wait is a block barrier
PB_D void mbar_init(uint64_t*, uint32_t) {}
PB_D void mbar_fence_init() {}
PB_D void mbar_expect_tx(uint64_t*, uint32_t) {}
PB_D void tma_bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t*) { memcpy(dst_smem, src_gmem, bytes); }
PB_D void mbar_wait(uint64_t*, uint32_t) { __syncthreads(); }
#define PB_DYNAMIC_SMEM(name) unsigned char* name = emu::g_dyn_smem
#else
#define PB_DYNAMIC_SMEM(name) extern __shared__ __align__(16) unsigned char name[]
PB_D void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
PB_D uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
PB_D void mbar_init(uint64_t* bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count)); }
PB_D void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
PB_D void tma_bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)), "l"(src_gmem),
                 "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
PB_D void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
#endif
// Stage `bytes` (multiple of 16, 16-byte aligned both sides) into shared memory; all threads return
// once the data has landed.
PB_D void stage_to_smem(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    if (threadIdx.x == 0) {
        mbar_init(bar, 1);
        mbar_fence_init();
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        mbar_expect_tx(bar, bytes);
        tma_bulk_g2s(dst, src, bytes, bar);
    }
    mbar_wait(bar, 0);
}

PB_D uint32_t warp_sum(uint32_t v) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
// warp-aggregated append: returns this lane's position in the output queue (valid when push)
PB_D uint32_t queue_append(uint32_t* counter, bool push) {
    unsigned m = __ballot_sync(0xffffffffu, push);
    uint32_t base = 0;
    int lane = threadIdx.x & 31;
    if (lane == 0 && m) base = atomicAdd(counter, (uint32_t)__popc(m));
    base = __shfl_sync(0xffffffffu, base, 0);
    return base + (uint32_t)__popc(m & ((1u << lane) - 1u));
}

struct BatchInfo {
    uint32_t first_pixel;   // linear pixel index (row-major inside rect) of the batch's first pixel
    uint32_t n_pixels;
    uint32_t first_sample;  // samples [first_sample, first_sample + n_samples) of each pixel
    uint32_t n_samples;
    uint64_t n_samples_magic;  // div_magic(., n_samples_magic) == . / n_samples (magic_of)
};

// A camera sample's path state: ray direction, beta = 1, Sobol' index, next dimension 5, for the dense layout of the fields.  The path
// integrator's interleaved record A is written by k_raygen's tail instead, whole and coalesced (see there).
PB_D void raygen_state(const DPaths& ps, uint32_t i, V3 d, uint64_t index) {
    if (ps.path_rec) return;
    ps.ray_d[i] = make_float4(d.x, d.y, d.z, 0.0f);
    ps.beta[i] = make_float4(1.0f, 1.0f, 1.0f, 1.0f);
    ps.sobol[i] = make_uint2((uint32_t)index, (uint32_t)(index >> 32));
    ps.dim[i] = 5u;
}

// k_raygen's slot for the realistic camera (integrator.rs:134-160): the camera sample's ray and weight.  A vignetted sample (weight 0)
// keeps a valid p_film and no PF_HAS_RAY: li does not run (L = 0), and k_resolve<true> still adds its filter weight to the pixel.
template <bool CAM_MOTION>
PB_D uint32_t raygen_lens(const DScene& sc, const DRender& rp, DPaths& ps, const DLens& lens, const DMotion& cam_mo, uint32_t i, uint64_t index, float2 p_film,
                          float time, float2 p_lens, float4& ray0, float4& ray1) {
    float c2w_t[16];
    if (CAM_MOTION) {
        float c2w_inv_t[16];
        motion_interpolate(cam_mo, lerpf(time, sc.shutter_open, sc.shutter_close), c2w_t, c2w_inv_t);
    }
    const float* c = CAM_MOTION ? c2w_t : sc.camera_to_world;
    V3 o, d, rxo, ryo, rxd, ryd;
    const float wt = lens_generate_ray_differential(lens, c, make_float2(sc.shutter_open, sc.shutter_close), p_film, p_lens, o, d, rxo, ryo, rxd, ryd);
    lens.weight[i] = wt;
    ps.p_film[i] = p_film;
    if (!(wt > 0.0f)) {  // integrator.rs:157: li only for ray_weight > 0
        ps.L[i] = make_float4(0.0f, 0.0f, 0.0f, __uint_as_float(0u));
        return 0;
    }
    if (ps.ray_diff) {  // scale_differentials(1 / sqrt(spp)) (integrator.rs:140-144)
        const float sdiff = 1.0f / sqrtf((float)rp.spp);
        rxo = o + (rxo - o) * sdiff;
        ryo = o + (ryo - o) * sdiff;
        rxd = d + (rxd - d) * sdiff;
        ryd = d + (ryd - d) * sdiff;
        ps.ray_diff[3 * (size_t)i] = make_float4(rxo.x, rxo.y, rxo.z, ryo.x);
        ps.ray_diff[3 * (size_t)i + 1] = make_float4(ryo.y, ryo.z, rxd.x, rxd.y);
        ps.ray_diff[3 * (size_t)i + 2] = make_float4(rxd.z, ryd.x, ryd.y, ryd.z);
    }
    ray0 = make_float4(o.x, o.y, o.z, __int_as_float(0x7f800000));
    ray1 = make_float4(d.x, d.y, d.z, __uint_as_float(i | (RAY_EXTEND << 30)));
    raygen_state(ps, i, d, index);
    ps.L[i] = make_float4(0.0f, 0.0f, 0.0f, __uint_as_float(PF_HAS_RAY));
    return 1;
}

// -----------------------------------------------------------------------------------------------
// Camera-sample Sobol' tables of one render (Sobol' sampler): 32-byte records {index lo, index hi, raw u32 of dims 0, 1}
// {raw u32 of dims 2, 3, 4, 0}, for
//   F[s] = I(s, 0, 0)   s < spp                        records [0, spp)
//   X[u] = I(0, u, 0)   u < sb[2] - sb[0]              records [spp, spp + wx)
//   Y[u] = I(0, 0, u)   u < sb[3] - sb[1]              records [spp + wx, spp + wx + wy)
// where I(s, x, y) = sobol_interval_to_index(m, s, x, y).  Every step of I is linear over GF(2):
//   I(s, x, y) = (s << 2m) ^ Lvdci(Lvdc(s) ^ (x << m | y)),  Lvdc / Lvdci(b) = XOR of the vdc / vdci rows over the set bits of b,
// the shifts drop bits past the word as a mask does, and y < 2^m makes x << m | y = (x << m) ^ y, so
//   I(s, x, y) = I(s, 0, 0) ^ I(0, x, 0) ^ I(0, 0, y).
// A dimension's raw u32 is the generator matrix applied to the index's first 4 * n_chunks bits, linear again, so it splits the same
// way.  k_raygen therefore XORs three records where it ran the bit loops of sobol_interval_to_index and five nibble-table walks, and
// gets the same bits.  The pixel coordinates relative to sb are below the sample bounds' extent (pixels lie in sb), itself <= 2^m.
__global__ void __launch_bounds__(256) k_camera_sobol(DRender rp, const uint32_t* __restrict__ nib, uint32_t n_chunks, const uint64_t* __restrict__ vdc,
                                                      const uint64_t* __restrict__ vdci, uint4* __restrict__ tab) {
    const uint32_t wx = (uint32_t)(rp.sb[2] - rp.sb[0]), wy = (uint32_t)(rp.sb[3] - rp.sb[1]);
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rp.spp + wx + wy) return;
    uint64_t frame = 0;
    int u = 0, v = 0;
    if (i < rp.spp) frame = i;
    else if (i < rp.spp + wx) u = (int)(i - rp.spp);
    else v = (int)(i - rp.spp - wx);
    const uint32_t m = rp.log2_res;  // (m == 0: every index is 0 and the rows are not read)
    const size_t row = m ? (size_t)(m - 1) * PB_SOBOL_MATRIX_SIZE : 0;
    SobolCtx sob;
    sob.nib = nib; sob.stride = PB_SOBOL_CHUNKS; sob.n_chunks = n_chunks; sob.dim = 0; sob.overflow = false;
    sob.index = sobol_interval_to_index(vdc + row, vdci + row, m, frame, u, v);
    tab[2 * (size_t)i] = make_uint4((uint32_t)sob.index, (uint32_t)(sob.index >> 32), sobol_sample_nib_u32(sob, 0), sobol_sample_nib_u32(sob, 1));
    tab[2 * (size_t)i + 1] = make_uint4(sobol_sample_nib_u32(sob, 2), sobol_sample_nib_u32(sob, 3), sobol_sample_nib_u32(sob, 4), 0u);
}
PB_D uint4 xor4(uint4 a, uint4 b) { return make_uint4(a.x ^ b.x, a.y ^ b.y, a.z ^ b.z, a.w ^ b.w); }

// -----------------------------------------------------------------------------------------------
// k_raygen: integrator.rs:123-144, sampler.rs:85-95, sobol.rs:110-138, and the camera's generate_ray_differential
// (perspective.rs:190-280, orthographic.rs:156-230, environment.rs:92-116).
// CAM_MOTION: the camera is animated (cam_mo); a static camera's instantiation never reads cam_mo.
// CAM_KIND: PbrtCameraKind.  env_res: Film.full_resolution as floats, read by the environment camera only.  lens: the realistic
// camera's lens system, pupil bounds and per-slot weight array, read by that camera only.  cam_sobol: this render's k_camera_sobol
// tables (Sobol' sampler; null for Halton).
template <bool CAM_MOTION, int CAM_KIND>
__global__ void __launch_bounds__(256) k_raygen(DScene sc, DRender rp, DPaths ps, BatchInfo bi, const uint4* __restrict__ cam_sobol, uint32_t* __restrict__ queue,
                                               uint32_t* __restrict__ d_count, float4* __restrict__ rays, uint32_t* __restrict__ d_nrays,
                                               DCounters* cnt, const DMotion cam_mo, const float2 env_res, const DLens lens) {
    constexpr bool ORTHO = CAM_KIND == PBRT_CAMERA_ORTHOGRAPHIC, ENV = CAM_KIND == PBRT_CAMERA_ENVIRONMENT, REAL = CAM_KIND == PBRT_CAMERA_REALISTIC;
    __shared__ uint32_t s_warp[8], s_base;  // the CTA's ray append (blockDim.x == 256)
    __shared__ float4 s_ray[256 * 2], s_rec[256 * 4];  // the CTA's rays and records A, staged for coalesced stores
    uint32_t n = bi.n_pixels * bi.n_samples;
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) *d_count = n;
    uint32_t my_rays = 0;
    float4 ray0 = make_float4(0.0f, 0.0f, 0.0f, 0.0f), ray1 = ray0;
    uint64_t ray_index = 0;  // the Sobol' / Halton index of the sample whose ray this thread made
    if (i < n) {
        const uint32_t pl = div_magic(i, bi.n_samples_magic), s = bi.first_sample + (i - pl * bi.n_samples);
        uint32_t pix = bi.first_pixel + pl;
        int px, py;
        const bool in_frame = share_pixel(rp, pix, px, py);
        queue[i] = i;
        bool inside = in_frame && px >= rp.pb[0] && px < rp.pb[2] && py >= rp.pb[1] && py < rp.pb[3];
        if (!inside) {  // integrator.rs:125-127: pixel skipped, no samples added
            ps.L[i] = make_float4(0.0f, 0.0f, 0.0f, __uint_as_float(0u));
            ps.p_film[i] = make_float2(__int_as_float(0x7fc00000), 0.0f);  // NaN marks "no sample"
        } else {
            uint64_t index;
            float sx, sy, time, lx, ly;
            if (rp.halton) {  // HaltonSampler: get_camera_sample draws dims 0..4 (sampler.rs:85-95); y of a 2D sample first
                index = halton_index(rp, px, py, (uint64_t)s);
                sy = halton_sample_dimension(rp, index, 1u);
                sx = halton_sample_dimension(rp, index, 0u);
                time = halton_sample_dimension(rp, index, 2u);
                ly = halton_sample_dimension(rp, index, 4u);
                lx = halton_sample_dimension(rp, index, 3u);
            } else {
                // index and raw dims 0..4 = F[s] ^ X[px - sb0] ^ Y[py - sb1] (k_camera_sobol)
                const uint4* f = cam_sobol + 2 * (size_t)s;
                const uint4* xr = cam_sobol + 2 * ((size_t)rp.spp + (uint32_t)(px - rp.sb[0]));
                const uint4* yr = cam_sobol + 2 * ((size_t)rp.spp + (uint32_t)(rp.sb[2] - rp.sb[0]) + (uint32_t)(py - rp.sb[1]));
                const uint4 a = xor4(xor4(__ldg(f), __ldg(xr)), __ldg(yr)), b = xor4(xor4(__ldg(f + 1), __ldg(xr + 1)), __ldg(yr + 1));
                index = (uint64_t)a.x | ((uint64_t)a.y << 32);
                // dims 0,1: film offset remapped to the pixel and clamped (sobol.rs:127-138)
                sx = sobol_to_float(a.z);
                sy = sobol_to_float(a.w);
                sx = sx * (float)rp.resolution + (float)rp.sb[0];
                sx = clampf(sx - (float)px, 0.0f, PB_ONE_MINUS_EPSILON);
                sy = sy * (float)rp.resolution + (float)rp.sb[1];
                sy = clampf(sy - (float)py, 0.0f, PB_ONE_MINUS_EPSILON);
                time = sobol_to_float(b.x);
                lx = sobol_to_float(b.y);
                ly = sobol_to_float(b.z);
            }
            float2 p_film = make_float2((float)px + sx, (float)py + sy);
            if constexpr (REAL) {  // realistic.rs:693-735 (pb_lens.cuh)
                my_rays = raygen_lens<CAM_MOTION>(sc, rp, ps, lens, cam_mo, i, index, p_film, time, make_float2(lx, ly), ray0, ray1);
                ray_index = index;
            } else {
                // raster -> camera (Transform::transform_point transform.rs:490-517)
                const float* m = sc.raster_to_camera;
                float x = p_film.x, y = p_film.y, z = 0.0f;
                float xp = m[0] * x + m[1] * y + m[2] * z + m[3];
                float yp = m[4] * x + m[5] * y + m[6] * z + m[7];
                float zp = m[8] * x + m[9] * y + m[10] * z + m[11];
                float wp = m[12] * x + m[13] * y + m[14] * z + m[15];
                V3 pc = mk3(xp, yp, zp);
                if (wp != 1.0f) { float inv = 1.0f / wp; pc = mk3(inv * xp, inv * yp, inv * zp); }
                V3 o = mk3(0.0f, 0.0f, 0.0f), d = norm3(pc);
                if (ORTHO) { o = pc; d = mk3(0.0f, 0.0f, 1.0f); }  // orthographic.rs:165-176
                if (ENV) {  // environment.rs:93-100 (f32 sin / cos: the glibc restatement)
                    const float theta = PB_PI * p_film.y / env_res.y, phi = 2.0f * PB_PI * p_film.x / env_res.x;
                    float st, ct, sp, cp;
                    sincos_rn(theta, st, ct);
                    sincos_rn(phi, sp, cp);
                    d = mk3(st * cp, ct, st * sp);
                }
                (void)time;  // ray.time only selects an animated transform; static cameras ignore it
                float c2w_t[16];
                if (CAM_MOTION) {  // AnimatedTransform::transform_ray (transform.rs:2114-2124) at ray.time = lerp(sample.time, shutter) (perspective.rs:226)
                    float c2w_inv_t[16];
                    motion_interpolate(cam_mo, lerpf(time, sc.shutter_open, sc.shutter_close), c2w_t, c2w_inv_t);
                }
                if (!ENV && sc.lens_radius > 0.0f) {  // (the same thin lens for the orthographic camera, orthographic.rs:177-188)
                    float2 pl2 = concentric_sample_disk(make_float2(lx, ly));
                    pl2 = make_float2(pl2.x * sc.lens_radius, pl2.y * sc.lens_radius);
                    float ft = sc.focal_distance / d.z;
                    V3 p_focus = o + d * ft;
                    o = mk3(pl2.x, pl2.y, 0.0f);
                    d = norm3(p_focus - o);
                }
                // camera -> world (Transform::transform_ray transform.rs:538-550, with origin error offset :662-708)
                const float* c = CAM_MOTION ? c2w_t : sc.camera_to_world;
                x = o.x; y = o.y; z = o.z;
                V3 ow = mk3(c[0] * x + c[1] * y + c[2] * z + c[3], c[4] * x + c[5] * y + c[6] * z + c[7], c[8] * x + c[9] * y + c[10] * z + c[11]);
                float wpc = c[12] * x + c[13] * y + c[14] * z + c[15];
                V3 o_err = mk3(fabsf(c[0] * x) + fabsf(c[1] * y) + fabsf(c[2] * z) + fabsf(c[3]), fabsf(c[4] * x) + fabsf(c[5] * y) + fabsf(c[6] * z) + fabsf(c[7]),
                               fabsf(c[8] * x) + fabsf(c[9] * y) + fabsf(c[10] * z) + fabsf(c[11])) * gamma_n(3);
                if (wpc != 1.0f) { float inv = 1.0f / wpc; ow = mk3(inv * ow.x, inv * ow.y, inv * ow.z); }
                V3 dw = mk3(c[0] * d.x + c[1] * d.y + c[2] * d.z, c[4] * d.x + c[5] * d.y + c[6] * d.z, c[8] * d.x + c[9] * d.y + c[10] * d.z);
                float ls = len2(dw);
                if (ls > 0.0f) {
                    float dt = dot3(abs3(dw), o_err) / ls;
                    ow = ow + dw * dt;
                }
                // textured scenes: the ray differential (perspective.rs:205-271), through camera_to_world (transform.rs:550-556), scaled
                // (integrator.rs:140-144).  The environment camera makes none (environment.rs:106).
                if (!ENV && ps.ray_diff) {
                    const V3 dxc = mk3(sc.dx_camera[0], sc.dx_camera[1], sc.dx_camera[2]), dyc = mk3(sc.dy_camera[0], sc.dy_camera[1], sc.dy_camera[2]);
                    V3 rxo = mk3(0.0f, 0.0f, 0.0f), ryo = rxo;
                    V3 rxd = norm3(pc + dxc), ryd = norm3(pc + dyc);
                    if (ORTHO) {  // orthographic.rs:189-226
                        rxo = o + dxc; ryo = o + dyc; rxd = d; ryd = d;
                        if (sc.lens_radius > 0.0f) {
                            // ft of the refracted ray.d, and one focus point (from dx_camera) for both differentials: ry == rx, as written
                            float2 pl2 = concentric_sample_disk(make_float2(lx, ly));
                            pl2 = make_float2(pl2.x * sc.lens_radius, pl2.y * sc.lens_radius);
                            const float ft = sc.focal_distance / d.z;
                            const V3 p_focus = pc + dxc + mk3(0.0f, 0.0f, 1.0f) * ft;
                            rxo = mk3(pl2.x, pl2.y, 0.0f); ryo = rxo;
                            rxd = norm3(p_focus - rxo); ryd = norm3(p_focus - ryo);
                        }
                    } else if (sc.lens_radius > 0.0f) {
                        float2 pl2 = concentric_sample_disk(make_float2(lx, ly));
                        pl2 = make_float2(pl2.x * sc.lens_radius, pl2.y * sc.lens_radius);
                        const V3 dx = norm3(pc + dxc);
                        const float ftx = sc.focal_distance / dx.z;
                        const V3 pfx = mk3(0.0f, 0.0f, 0.0f) + dx * ftx;
                        rxo = mk3(pl2.x, pl2.y, 0.0f);
                        rxd = norm3(pfx - rxo);
                        const V3 dy = norm3(pc + dyc);
                        const float fty = sc.focal_distance / dy.z;
                        const V3 pfy = mk3(0.0f, 0.0f, 0.0f) + dy * fty;
                        ryo = mk3(pl2.x, pl2.y, 0.0f);
                        ryd = norm3(pfy - ryo);
                    }
                    auto xp = [c](V3 q) {
                        V3 r = mk3(c[0] * q.x + c[1] * q.y + c[2] * q.z + c[3], c[4] * q.x + c[5] * q.y + c[6] * q.z + c[7], c[8] * q.x + c[9] * q.y + c[10] * q.z + c[11]);
                        const float w = c[12] * q.x + c[13] * q.y + c[14] * q.z + c[15];
                        if (w != 1.0f) { const float inv = 1.0f / w; r = mk3(inv * r.x, inv * r.y, inv * r.z); }
                        return r;
                    };
                    auto xv = [c](V3 v) { return mk3(c[0] * v.x + c[1] * v.y + c[2] * v.z, c[4] * v.x + c[5] * v.y + c[6] * v.z, c[8] * v.x + c[9] * v.y + c[10] * v.z); };
                    rxo = xp(rxo); ryo = xp(ryo); rxd = xv(rxd); ryd = xv(ryd);
                    const float sdiff = 1.0f / sqrtf((float)rp.spp);
                    rxo = ow + (rxo - ow) * sdiff;
                    ryo = ow + (ryo - ow) * sdiff;
                    rxd = dw + (rxd - dw) * sdiff;
                    ryd = dw + (ryd - dw) * sdiff;
                    ps.ray_diff[3 * (size_t)i] = make_float4(rxo.x, rxo.y, rxo.z, ryo.x);
                    ps.ray_diff[3 * (size_t)i + 1] = make_float4(ryo.y, ryo.z, rxd.x, rxd.y);
                    ps.ray_diff[3 * (size_t)i + 2] = make_float4(rxd.z, ryd.x, ryd.y, ryd.z);
                }
                ray0 = make_float4(ow.x, ow.y, ow.z, __int_as_float(0x7f800000));  // t_max = inf - dt = inf
                ray1 = make_float4(dw.x, dw.y, dw.z, __uint_as_float(i | (RAY_EXTEND << 30)));
                raygen_state(ps, i, dw, index);
                ps.L[i] = make_float4(0.0f, 0.0f, 0.0f, __uint_as_float(PF_HAS_RAY));
                ps.p_film[i] = p_film;
                my_rays = 1;
                ray_index = index;
            }
        }
    }
    // One append per CTA: a ray's place in the queue is not observable in the results.  A warp's rays are contiguous in the queue and
    // its 32 records A in the path state, so both are staged in shared memory and stored 512 contiguous bytes per instruction rather
    // than one 16-byte piece of a different record per lane.  Record A is written whole, its unused first 16 bytes and last word
    // included: the L2 writes back a partly written 32-byte sector only after reading the rest of it from HBM.  (A slot without a ray
    // gets a record too; nothing reads it.)
    const unsigned bal = __ballot_sync(0xffffffffu, my_rays != 0);
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    if (lane == 0) s_warp[warp] = (uint32_t)__popc(bal);
    if (my_rays) {
        const uint32_t k = 2u * (32u * warp + (uint32_t)__popc(bal & ((1u << lane) - 1u)));
        s_ray[k] = ray0;
        s_ray[k + 1] = ray1;
    }
    if (ps.path_rec) {
        const float4 z = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        float4* r = s_rec + 4 * threadIdx.x;
        r[0] = z;
        r[1] = my_rays ? make_float4(ray1.x, ray1.y, ray1.z, 0.0f) : z;
        r[2] = make_float4(1.0f, 1.0f, 1.0f, 1.0f);
        r[3] = my_rays ? make_float4(__uint_as_float((uint32_t)ray_index), __uint_as_float((uint32_t)(ray_index >> 32)), __uint_as_float(5u), 0.0f) : z;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t tot = 0;
        for (int w = 0; w < 8; ++w) { const uint32_t c = s_warp[w]; s_warp[w] = tot; tot += c; }
        s_base = tot ? atomicAdd(d_nrays, tot) : 0u;  // *d_nrays is zeroed by the host before the launch
        if (tot) atomicAdd(&cnt->camera_rays, (unsigned long long)tot);
    }
    __syncthreads();
    const size_t wpos = s_base + s_warp[warp];
    for (uint32_t k = lane; k < 2u * (uint32_t)__popc(bal); k += 32u) rays[2 * wpos + k] = s_ray[64u * warp + k];
    if (ps.path_rec) {
        const uint32_t first = blockIdx.x * blockDim.x + 32u * warp;  // this warp's first slot
        for (uint32_t k = lane; k < 128u; k += 32u)
            if (first + (k >> 2) < n) ps.path_rec[4 * (size_t)first + k] = s_rec[128u * warp + k];
    }
}

// -----------------------------------------------------------------------------------------------
// Light-grid voxel of a point (lightdistrib.rs:282-294)
PB_D uint32_t light_voxel(const DScene& sc, const DLightGrid& g, V3 p) {
    float ox = p.x - sc.wb_min[0], oy = p.y - sc.wb_min[1], oz = p.z - sc.wb_min[2];
    if (sc.wb_max[0] > sc.wb_min[0]) ox = fdiv0(ox, sc.wb_max[0] - sc.wb_min[0]);  // points on the bound's min faces: 0 / extent
    if (sc.wb_max[1] > sc.wb_min[1]) oy = fdiv0(oy, sc.wb_max[1] - sc.wb_min[1]);
    if (sc.wb_max[2] > sc.wb_min[2]) oz = fdiv0(oz, sc.wb_max[2] - sc.wb_min[2]);
    int ix = min(max(f2i_sat(ox * (float)g.nv[0]), 0), g.nv[0] - 1);
    int iy = min(max(f2i_sat(oy * (float)g.nv[1]), 0), g.nv[1] - 1);
    int iz = min(max(f2i_sat(oz * (float)g.nv[2]), 0), g.nv[2] - 1);
    return ((uint32_t)iz * (uint32_t)g.nv[1] + (uint32_t)iy) * (uint32_t)g.nv[0] + (uint32_t)ix;
}

// -----------------------------------------------------------------------------------------------
// k_trace: Scene::intersect (scene.rs:55) / Scene::intersect_p (scene.rs:67) for every record of the ray
// queue.  Persistent: the grid is sized to the resident CTAs of the device and warps pull rays until the
// queue is empty (pb_trace.cuh::trace_rays).  When the whole BVH + triangle list fits in shared memory
// (Cornell-class scenes) it is staged there once per CTA by a TMA bulk copy.
// The alpha tests of Triangle::intersect / intersect_p for a candidate hit (declared in pb_trace.cuh): the local interaction carries
// p_hit and uv_hit and no differentials -- all a texture lookup reads --, intersect_p first runs its own dpdu / dpdv block, which
// rejects a degenerate triangle (triangle.rs:594-627).  true = the candidate is rejected.
__device__ PB_NOINLINE bool alpha_rejects(const DScene& sc, uint32_t prim, V3 p0, V3 p1, V3 p2, float b0, float b1, float b2, uint32_t flags, bool any_hit) {
    const uint4 idx = __ldg(sc.tri_idx + prim);
    float2 uv0 = make_float2(0.0f, 0.0f), uv1 = make_float2(1.0f, 0.0f), uv2 = make_float2(1.0f, 1.0f);  // triangle.rs:96-110
    if (flags & TRI_HAS_UV) {
        uv0 = make_float2(__ldg(sc.vuv + 2 * (size_t)idx.x), __ldg(sc.vuv + 2 * (size_t)idx.x + 1));
        uv1 = make_float2(__ldg(sc.vuv + 2 * (size_t)idx.y), __ldg(sc.vuv + 2 * (size_t)idx.y + 1));
        uv2 = make_float2(__ldg(sc.vuv + 2 * (size_t)idx.z), __ldg(sc.vuv + 2 * (size_t)idx.z + 1));
    }
    if (any_hit) {
        const float duv02x = uv0.x - uv2.x, duv02y = uv0.y - uv2.y, duv12x = uv1.x - uv2.x, duv12y = uv1.y - uv2.y;
        const V3 dp02 = p0 - p2, dp12 = p1 - p2;
        const float determinant = duv02x * duv12y - duv02y * duv12x;
        const bool degenerate_uv = fabsf(determinant) < 1e-8f;
        V3 dpdu = mk3(0.0f, 0.0f, 0.0f), dpdv = mk3(0.0f, 0.0f, 0.0f);
        if (!degenerate_uv) {
            const float invdet = 1.0f / determinant;
            dpdu = (dp02 * duv12y - dp12 * duv02y) * invdet;
            dpdv = (dp02 * -duv12x + dp12 * duv02x) * invdet;
        }
        if ((degenerate_uv || len2(cross3(dpdu, dpdv)) == 0.0f) && len2(cross3(p2 - p0, p1 - p0)) == 0.0f) return true;  // "the intersection is bogus"
    }
    Isect is;
    is.p = p0 * b0 + p1 * b1 + p2 * b2;
    is.uv = make_float2(uv0.x * b0 + uv1.x * b1 + uv2.x * b2, uv0.y * b0 + uv1.y * b1 + uv2.y * b2);
    UvDiff dd;
    dd.dudx = dd.dvdx = dd.dudy = dd.dvdy = 0.0f;
    dd.dpdx = dd.dpdy = mk3(0.0f, 0.0f, 0.0f);
    const uint2 ma = __ldg(sc.mesh_alpha + idx.w);
    if ((flags & TRI_ALPHA) && texture_evaluate(sc.textures, ma.x - 1u, sc.ewa_lut, is, dd).r == 0.0f) return true;
    if (any_hit && (flags & TRI_SHADOW_ALPHA) && texture_evaluate(sc.textures, ma.y - 1u, sc.ewa_lut, is, dd).r == 0.0f) return true;
    return false;
}

template <bool COUNT, int MODE, bool SMEM, bool INST = false, bool ALPHA = false>
__global__ void __launch_bounds__(PB_TRACE_THREADS) k_trace(DScene sc, TraceIO io, const uint32_t* __restrict__ d_nrays, uint32_t n_rays_host,
                                                          uint32_t* __restrict__ cursor, DCounters* cnt) {
    PB_DYNAMIC_SMEM(smem_raw);
    __shared__ __align__(8) uint64_t s_bar;
    const float4* nodes = sc.nodes;
    const float4* tris = sc.tri_verts;
    if (SMEM) {
        const uint32_t nb = sc.n_nodes * 32u, tb = sc.n_tris * 48u;
        if (threadIdx.x == 0) {
            mbar_init(&s_bar, 1);
            mbar_fence_init();
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            mbar_expect_tx(&s_bar, nb + tb);
            tma_bulk_g2s(smem_raw, sc.nodes, nb, &s_bar);
            tma_bulk_g2s(smem_raw + nb, sc.tri_verts, tb, &s_bar);
        }
        mbar_wait(&s_bar, 0);
        nodes = reinterpret_cast<const float4*>(smem_raw);
        tris = reinterpret_cast<const float4*>(smem_raw + nb);
    }
    const uint32_t n_rays = d_nrays ? *d_nrays : n_rays_host;
    trace_rays<COUNT, MODE, SMEM, INST, ALPHA>(sc, nodes, tris, io, n_rays, cursor, cnt);
}

// k_flatten_tris (pbrt_gpu_scene_create): the caller's PbrtTri records -> the pre-gathered 48-byte triangle records and the per-triangle
// attribute indices, one thread per triangle, with the index checks the host used to make while flattening (status[0] = the largest
// error code met, 0 = fine; status[1] = some triangle has Material "none").  tris: PbrtTri as 3 x uint2 {v0, v1} {v2, mesh} {material, area_light}.
struct DMeshRec { uint32_t vbase, n_verts, flags, pad; };
__global__ void __launch_bounds__(256) k_flatten_tris(const uint2* __restrict__ tris, uint32_t n_tris, const DMeshRec* __restrict__ meshes, uint32_t n_meshes,
                                                     const float* __restrict__ vp, uint32_t n_materials, uint32_t n_lights, uint32_t n_instances,
                                                     float4* __restrict__ tv, uint4* __restrict__ tidx, uint32_t* __restrict__ status) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_tris) return;
    const uint2 a = tris[3 * (size_t)i], b = tris[3 * (size_t)i + 1], c = tris[3 * (size_t)i + 2];
    const uint32_t v0 = a.x, v1 = a.y, v2 = b.x, mesh = b.y, material = c.x;
    const int area_light = (int)c.y;
    uint32_t err = 0;
    if (mesh == 0xffffffffu) {  // PBRT_MESH_INSTANCE: a TransformedPrimitive, the record only names the instance
        if (v0 >= n_instances) err = 5;
        else {
            tv[3 * (size_t)i] = make_float4(__uint_as_float(v0), 0.0f, 0.0f, 0.0f);
            tv[3 * (size_t)i + 1] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
            tv[3 * (size_t)i + 2] = make_float4(0.0f, __uint_as_float(0xffffffffu), __uint_as_float(0xffffffffu), __uint_as_float((uint32_t)TRI_INSTANCE));
            tidx[i] = make_uint4(0, 0, 0, 0);
        }
    } else if (mesh >= n_meshes) err = 1;
    else {
        const DMeshRec m = meshes[mesh];
        if (v0 >= m.n_verts || v1 >= m.n_verts || v2 >= m.n_verts) err = 2;
        else if (material != 0xffffffffu && material >= n_materials) err = 3;
        else if (area_light >= (int)n_lights) err = 4;
        else if (area_light >= 0 && (m.flags & (TRI_ALPHA | TRI_SHADOW_ALPHA))) err = 6;
        else {
            if (material == 0xffffffffu) status[1] = 1u;
            const float* p0 = vp + 3 * (size_t)(m.vbase + v0);
            const float* p1 = vp + 3 * (size_t)(m.vbase + v1);
            const float* p2 = vp + 3 * (size_t)(m.vbase + v2);
            tv[3 * (size_t)i] = make_float4(p0[0], p0[1], p0[2], p1[0]);
            tv[3 * (size_t)i + 1] = make_float4(p1[1], p1[2], p2[0], p2[1]);
            tv[3 * (size_t)i + 2] = make_float4(p2[2], __uint_as_float(material), __uint_as_float((uint32_t)area_light), __uint_as_float(m.flags));
            tidx[i] = make_uint4(m.vbase + v0, m.vbase + v1, m.vbase + v2, mesh);
        }
    }
    if (err) atomicMax(status, err);
}

// k_wide_build: the wide records of trace_rays_wide from the reference-layout node array, one thread per node (leaves own no record:
// their primitive range is carried by the parent's child reference).
__global__ void __launch_bounds__(256) k_wide_build(const float4* __restrict__ nodes, uint32_t n_nodes, float4* __restrict__ wide) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_nodes) return;
    const float4 m1 = nodes[2 * (size_t)i + 1];
    const uint32_t meta = __float_as_uint(m1.w);
    if (meta & 0xffffu) return;  // a leaf
    const uint32_t c[2] = {i + 1u, __float_as_uint(m1.z)};  // first child follows its parent, second child at `offset` (bvh.rs:393-400)
    float4 a[2], b[2];
    uint32_t ref[2];
    for (int k = 0; k < 2; ++k) {
        a[k] = nodes[2 * (size_t)c[k]];
        b[k] = nodes[2 * (size_t)c[k] + 1];
        const uint32_t cm = __float_as_uint(b[k].w), np = cm & 0xffffu;
        ref[k] = np ? (__float_as_uint(b[k].z) | (np << PB_WIDE_LEAF_SHIFT)) : c[k];
    }
    float4* o = wide + 4 * (size_t)i;
    o[0] = make_float4(a[0].x, a[0].y, a[0].z, a[0].w);
    o[1] = make_float4(b[0].x, b[0].y, a[1].x, a[1].y);
    o[2] = make_float4(a[1].z, a[1].w, b[1].x, b[1].y);
    o[3] = make_float4(__uint_as_float(ref[0]), __uint_as_float(ref[1]), __uint_as_float((meta >> 16) & 3u), 0.0f);
}
// Launch bounds of the wide trace kernels.  Plain scenes: NO minimum-CTA bound -- ptxas then settles on 64 registers (8 CTAs of 128
// threads per SM), which beat a bound of 1, a bound of 8 (registers squeezed), and 9 or 10 CTAs with the leaf-only ray state in shared
// memory (48 registers at 10): those were slower at every L1 size tried, including the same 92 KB of L1 (DESIGN.md §7, §9).
// PB_WIDE_MIN_BLOCKS > 0 sets a bound for experiments.  Instanced scenes: a bound of 8 (64 registers instead of 80) was the faster choice on the landscape.
#ifndef PB_WIDE_MIN_BLOCKS
#define PB_WIDE_MIN_BLOCKS 0
#endif
#ifndef PB_WIDE_INST_MIN_BLOCKS
#define PB_WIDE_INST_MIN_BLOCKS 8
#endif
#if PB_WIDE_MIN_BLOCKS > 0
#define PB_WIDE_BOUNDS __launch_bounds__(PB_TRACE_THREADS, PB_WIDE_MIN_BLOCKS)
#else
#define PB_WIDE_BOUNDS __launch_bounds__(PB_TRACE_THREADS)
#endif
__global__ void PB_WIDE_BOUNDS k_trace_wide_plain(DScene sc, TraceIO io, const uint32_t* __restrict__ d_nrays, uint32_t* __restrict__ cursor, DCounters* cnt, int walk_steps) {
    trace_rays_wide<false>(sc, sc.wide, sc.tri_verts, io, *d_nrays, cursor, cnt, walk_steps);
}
__global__ void __launch_bounds__(PB_TRACE_THREADS, PB_WIDE_INST_MIN_BLOCKS) k_trace_wide_inst(DScene sc, TraceIO io, const uint32_t* __restrict__ d_nrays, uint32_t* __restrict__ cursor,
                                                                                             DCounters* cnt, int walk_steps) {
    trace_rays_wide<true>(sc, sc.wide, sc.tri_verts, io, *d_nrays, cursor, cnt, walk_steps);
}

__global__ void PB_WIDE_BOUNDS k_trace_wide_spec(DScene sc, TraceIO io, const uint32_t* __restrict__ d_nrays,
                                                                                        uint32_t* __restrict__ cursor, DCounters* cnt, int walk_steps) {
    trace_rays_wide_spec(sc, sc.wide, sc.tri_verts, io, *d_nrays, cursor, cnt, walk_steps);
}

// k_rayprep: the per-ray constants of the traversal and of the watertight triangle test (pb_trace.cuh::make_ray: reciprocal direction,
// permutation, shear) for every record of the ray queue, one thread per ray, fully coalesced; k_trace's lanes then load them
// instead of recomputing them when they fetch a ray.  Same arithmetic, so nothing a ray reports changes.
__global__ void __launch_bounds__(256) k_rayprep(const float4* __restrict__ rays, const uint32_t* __restrict__ d_nrays, float4* __restrict__ pre) {
    const uint32_t n = *d_nrays;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const float4 a = rays[2 * (size_t)i], b = rays[2 * (size_t)i + 1];
        const RayPre r = make_ray(mk3(a.x, a.y, a.z), mk3(b.x, b.y, b.z));
        float4 p0, p1;
        pack_ray(r, p0, p1);
        pre[2 * (size_t)i] = p0;
        pre[2 * (size_t)i + 1] = p1;
    }
}

// k_sort: everything the traced rays leave to do before the next surface is shaded, then the bucketing of those surface hits for
// k_shade.  First the previous vertex's estimate_direct is finished with the shadow / MIS results (integrator.rs:461-567), then a path
// ray that escaped adds the environment emission (path.rs:267-275): the reference adds both before the Le of the next vertex, so they
// come first here too.  A slot without a surface hit is then finished -- L is final, its flags are 0 -- and joins no queue.  A hit goes
// to class c >= 1, the shading class of its material (same lobe-kind sequence => same code path; warp match + prefix sum); null-
// material hits go to class 1.  Also raises the spatial light distribution's voxel requests for the hits
// (the lookup of path.rs:118; extra requests are harmless, the distribution of a voxel is deterministic).
// The counters the NEXT kernels append to are reset here rather than by memsets between the launches (five per iteration before):
// k_sort clears the survivor count and the ray count k_shade is about to fill, k_shade clears what the next iteration's k_trace /
// k_sort fill (ray cursor, voxel requests, the other set of class counts).
__global__ void __launch_bounds__(256) k_sort(DScene sc, DPaths ps, DLightGrid grid, uint32_t spatial, uint32_t instancing, const uint32_t* __restrict__ queue,
                                             const uint32_t* __restrict__ d_count, uint32_t* __restrict__ cls_queue, uint32_t cls_stride,
                                             uint32_t* __restrict__ cls_count, uint32_t* __restrict__ reset_count_out, uint32_t* __restrict__ reset_nrays) {
    if (blockIdx.x == 0 && threadIdx.x == 0) { *reset_count_out = 0u; *reset_nrays = 0u; }
    const uint32_t count = *d_count;
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t total = (count + 31u) & ~31u;
    for (uint32_t qi = blockIdx.x * blockDim.x + threadIdx.x; qi < total; qi += gridDim.x * blockDim.x) {
        uint32_t cls = 0xffffffffu, slot = 0;
        if (qi < count) {
            slot = queue[qi];
            const float4 Lf = ps.L[slot];
            const uint32_t flags = __float_as_uint(Lf.w);
            Sp L = mksp(Lf.x, Lf.y, Lf.z);
            if (flags & (PF_HAS_SHADOW | PF_HAS_MIS)) {  // the next-event estimate of the previous vertex
                Sp ld = sp1(0.0f);
                const float4 a = ps.ld_light[slot];
                if ((flags & PF_HAS_SHADOW) && ps.occl[slot] == 0u) ld = ld + mksp(a.x, a.y, a.z);
                if (flags & PF_HAS_MIS) {
                    const float4 mh = ps.mis_hit[slot];
                    int mprim = __float_as_int(mh.x);
                    if (mprim >= 0) {
                        const float4 md = ps.mis_d[slot], mf = ps.mis_f[slot];
                        int light_num = (int)__float_as_uint(md.w);
                        V3 lp, ln;
                        int hit_light;
                        tri_point_normal(sc, (uint32_t)mprim, mh.y, mh.z, mh.w, lp, ln, hit_light);
                        if (hit_light == light_num) {
                            Sp le = light_L(sc.lights[light_num], ln, -mk3(md.x, md.y, md.z));
                            if (!is_black(le)) ld = ld + mksp(mf.x, mf.y, mf.z) * le * sp1(1.0f) * a.w / mf.w;
                        }
                    } else if (sc.n_inf) {  // the MIS ray left the scene: li = light.le(ray) (integrator.rs:560-562)
                        const float4 md = ps.mis_d[slot], mf = ps.mis_f[slot];
                        Sp le = light_le(sc, sc.lights[__float_as_uint(md.w)], mk3(md.x, md.y, md.z));
                        if (!is_black(le)) ld = ld + mksp(mf.x, mf.y, mf.z) * le * sp1(1.0f) * a.w / mf.w;
                    }
                }
                const float4 nb = ps.nee_beta[slot];
                L = L + mksp(nb.x, nb.y, nb.z) * spdiv0(ld, nb.w);  // ld is black for every occluded light sample
            }
            if (flags & PF_HAS_RAY) {
                float4 h = ps.hit[slot];
                int prim = __float_as_int(h.x);
                if (prim < 0) {
                    // the path ray escaped: environment emission (path.rs:267-275)
                    if (sc.n_inf && ((flags >> PF_BOUNCES_SHIFT) == 0 || (flags & PF_SPECULAR_BOUNCE))) {
                        const float4 b4 = ps.beta[slot], rd4 = ps.ray_d[slot];
                        const Sp beta = mksp(b4.x, b4.y, b4.z);
                        const V3 rd = mk3(rd4.x, rd4.y, rd4.z);
                        for (uint32_t k = 0; k < sc.n_inf; ++k) L = L + beta * light_le(sc, sc.lights[sc.inf[k]], rd);
                    }
                } else {
                    float4 c = __ldg(sc.tri_verts + 3 * (size_t)prim + 2);
                    uint32_t mat = __float_as_uint(c.y);
                    const uint32_t inst = sc.n_instances ? ps.hit_inst[slot] : 0xffffffffu;
                    const bool moved = inst != 0xffffffffu && !sc.instances[inst].identity;
                    if (moved && instancing == 0u) mat = 0xffffffffu;  // the transformed interaction lost its primitive (quirk Q7)
                    cls = (mat == 0xffffffffu) ? 1u : ((uint32_t)sc.materials[mat].cls & 0xffu);
                    if (spatial) {
                        float4 a = __ldg(sc.tri_verts + 3 * (size_t)prim), b = __ldg(sc.tri_verts + 3 * (size_t)prim + 1);
                        V3 p = mk3(a.x, a.y, a.z) * h.y + mk3(a.w, b.x, b.y) * h.z + mk3(b.z, b.w, c.x) * h.w;
                        if (moved) {  // isect.p in world space (Transform::transform_point_with_abs_error's point)
                            const float* m = sc.instances[inst].m;
                            const float xp = m[0] * p.x + m[1] * p.y + m[2] * p.z + m[3], yp = m[4] * p.x + m[5] * p.y + m[6] * p.z + m[7];
                            const float zp = m[8] * p.x + m[9] * p.y + m[10] * p.z + m[11], wp = m[12] * p.x + m[13] * p.y + m[14] * p.z + m[15];
                            p = mk3(xp, yp, zp);
                            if (wp != 1.0f) { const float inv = 1.0f / wp; p = mk3(inv * xp, inv * yp, inv * zp); }
                        }
                        uint32_t v = light_voxel(sc, grid, p);
                        if (grid.state[v] == 0 && atomicCAS(&grid.state[v], 0, 1) == 0) {
                            if (grid.row) {  // sparse tables: the voxel's row is handed out with the request
                                uint32_t r = atomicAdd(grid.n_request + 1, 1u);
                                if (r >= grid.max_rows) { r = 0u; atomicOr(grid.n_request + 2, 1u); }  // the host fails the render
                                grid.row[v] = (int)r;
                            }
                            grid.request[atomicAdd(grid.n_request, 1u)] = v;
                        }
                    }
                }
            }
            if (cls == 0xffffffffu) ps.L[slot] = make_float4(L.r, L.g, L.b, __uint_as_float(0u));
            else if (flags & (PF_HAS_SHADOW | PF_HAS_MIS)) ps.L[slot] = make_float4(L.r, L.g, L.b, __uint_as_float(flags & ~(PF_HAS_SHADOW | PF_HAS_MIS)));
        }
        // one atomic per distinct class in the warp
        unsigned peers = __match_any_sync(0xffffffffu, cls);
        uint32_t base = 0;
        int leader = __ffs(peers) - 1;
        if (cls != 0xffffffffu && (int)lane == leader) base = atomicAdd(cls_count + cls, (uint32_t)__popc(peers));
        base = __shfl_sync(0xffffffffu, base, leader);
        if (cls != 0xffffffffu) cls_queue[(size_t)cls * cls_stride + base + (uint32_t)__popc(peers & ((1u << lane) - 1u))] = slot;
    }
}

// -----------------------------------------------------------------------------------------------
// SpatialLightDistribution::compute_distribution (lightdistrib.rs:169-269), split in two kernels:
// one thread per (requested voxel, light) accumulates the 128 Halton samples IN ORDER, then one
// thread per voxel builds the Distribution1D (sampling.rs:24-49).
template <int LIGHTS>
__global__ void k_lightgrid_contrib(DScene sc, DLightGrid g, const float* __restrict__ halton /* 128 x 5 */) {
    uint32_t nreq = *g.n_request;
    uint32_t total = nreq * (uint32_t)g.n_lights;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        uint32_t v = g.request[i / (uint32_t)g.n_lights], j = i % (uint32_t)g.n_lights;
        int ix = (int)(v % (uint32_t)g.nv[0]), iy = (int)((v / (uint32_t)g.nv[0]) % (uint32_t)g.nv[1]), iz = (int)(v / ((uint32_t)g.nv[0] * (uint32_t)g.nv[1]));
        float t0x = (float)ix / (float)g.nv[0], t0y = (float)iy / (float)g.nv[1], t0z = (float)iz / (float)g.nv[2];
        float t1x = (float)(ix + 1) / (float)g.nv[0], t1y = (float)(iy + 1) / (float)g.nv[1], t1z = (float)(iz + 1) / (float)g.nv[2];
        V3 vmin = mk3(lerpf(t0x, sc.wb_min[0], sc.wb_max[0]), lerpf(t0y, sc.wb_min[1], sc.wb_max[1]), lerpf(t0z, sc.wb_min[2], sc.wb_max[2]));
        V3 vmax = mk3(lerpf(t1x, sc.wb_min[0], sc.wb_max[0]), lerpf(t1y, sc.wb_min[1], sc.wb_max[1]), lerpf(t1z, sc.wb_min[2], sc.wb_max[2]));
        const DLight& light = sc.lights[j];
        float contrib = 0.0f;
        for (int s = 0; s < 128; ++s) {
            const float* hs = halton + 5 * s;
            V3 po = mk3(lerpf(__ldg(hs), vmin.x, vmax.x), lerpf(__ldg(hs + 1), vmin.y, vmax.y), lerpf(__ldg(hs + 2), vmin.z, vmax.z));
            float pdf = 0.0f;
            V3 wi;
            LightSample ls;
            Sp li = light_sample_li<LIGHTS>(sc, light, po, make_float2(__ldg(hs + 3), __ldg(hs + 4)), wi, pdf, ls);
            if (pdf > 0.0f) contrib += lum(li) / pdf;
        }
        g.contrib[g.row_of(v) * g.n_lights + j] = contrib;
    }
}
__global__ void k_lightgrid_build(DLightGrid g) {
    uint32_t nreq = *g.n_request;
    const int nl = g.n_lights;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < nreq; i += gridDim.x * blockDim.x) {
        uint32_t v = g.request[i];
        const size_t r = g.row_of(v);
        const float* c = g.contrib + r * nl;
        float sum = 0.0f;
        for (int j = 0; j < nl; ++j) sum += c[j];
        float avg = sum / (float)(128 * nl);
        float min_contrib = (avg > 0.0f) ? 0.001f * avg : 1.0f;
        float* func = g.func + r * nl;
        float* cdf = g.cdf + r * (nl + 1);
        cdf[0] = 0.0f;
        for (int j = 0; j < nl; ++j) {
            float f = fmaxf(c[j], min_contrib);
            func[j] = f;
            cdf[j + 1] = cdf[j] + f / (float)nl;
        }
        float func_int = cdf[nl];
        if (func_int == 0.0f) for (int j = 1; j <= nl; ++j) cdf[j] = (float)j / (float)nl;
        else for (int j = 1; j <= nl; ++j) cdf[j] /= func_int;
        g.func_int[r] = func_int;
        __threadfence();
        g.state[v] = 2;
    }
}

// Distribution1D::sample_discrete (sampling.rs:103-141)
PB_D int sample_discrete(const float* __restrict__ func, const float* __restrict__ cdf, float func_int, int n, float u, float& pdf) {
    // find_interval's result is the number of leading cdf entries that are <= u (the cdf is non-decreasing: running sums of
    // non-negative terms, then divided by their positive total), so any search order finds the same `first`.  With many lights the
    // reference's binary search is eight dependent loads per vertex from a table row nobody else in the warp shares; here one round of
    // independent loads picks a 16-entry bucket and a second one counts inside it.
    int first = 0;
    if (n >= 32) {
        const int nb = (n + 1 + 15) >> 4;  // buckets of 16 entries over cdf[0 .. n]
        int b = 0;
        for (int k = 1; k < nb; ++k) b += (cdf[16 * k] <= u) ? 1 : 0;  // entries 16, 32, ...: bucket = how many bucket heads are <= u
        const int lo = 16 * b, hi = min(lo + 16, n + 1);
        first = lo;
        for (int j = lo; j < hi; ++j) first += (cdf[j] <= u) ? 1 : 0;
    } else {
        int len = n + 1;
        while (len > 0) {
            int half = len >> 1, middle = first + half;
            if (cdf[middle] <= u) { first = middle + 1; len -= half + 1; }
            else len = half;
        }
    }
    int off = min(max(first - 1, 0), n - 1);
    pdf = (func_int > 0.0f) ? func[off] / (func_int * (float)n) : 0.0f;
    return off;
}

// -----------------------------------------------------------------------------------------------
// Ray coherence order.  k_shade appends rays in shading order, which after the first bounce is unrelated to where the rays
// go.  k_shade therefore emits a 13-bit key per ray (any-hit?, direction octant, 8x8x8 origin cell of the world bound) next to
// the ray record, and three small kernels turn the keys into a permutation (counting sort over 8192 keys, 4 B read + 4 B
// written per ray and pass); k_trace pulls rays through it, so the lanes of a warp walk the same part of the BVH (fewer
// divergent node/leaf phases).  Every ray is traced exactly as before: the order of a ray queue is not observable.
#define PB_RAY_KEYS 8192
PB_D uint32_t ray_key(const DScene& sc, const float4 a, const float4 b) {
    const uint32_t oct = (b.x < 0.0f ? 1u : 0u) | (b.y < 0.0f ? 2u : 0u) | (b.z < 0.0f ? 4u : 0u);
    const uint32_t shadow = (__float_as_uint(b.w) >> 30) == RAY_SHADOW ? 1u : 0u;
    uint32_t cell = 0;
    const float o[3] = {a.x, a.y, a.z};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float e = sc.wb_max[k] - sc.wb_min[k];
        int c = e > 0.0f ? (int)((o[k] - sc.wb_min[k]) / e * 8.0f) : 0;
        c = c < 0 ? 0 : (c > 7 ? 7 : c);
        cell = (cell << 3) | (uint32_t)c;
    }
    return (shadow << 12) | (oct << 9) | cell;
}
__global__ void __launch_bounds__(256) k_ray_hist(const uint32_t* __restrict__ d_nrays, const uint32_t* __restrict__ keys, uint32_t* __restrict__ hist) {
    __shared__ uint32_t s_hist[PB_RAY_KEYS];
    for (uint32_t i = threadIdx.x; i < PB_RAY_KEYS; i += blockDim.x) s_hist[i] = 0;
    __syncthreads();
    const uint32_t n = *d_nrays;
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t total = (n + 31u) & ~31u;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const uint32_t k = i < n ? keys[i] : 0xffffffffu;
        // neighbouring rays mostly share their key: one shared-memory atomic per distinct key of the warp
        const unsigned peers = __match_any_sync(0xffffffffu, k);
        if (k != 0xffffffffu && (int)lane == __ffs(peers) - 1) atomicAdd(&s_hist[k], (uint32_t)__popc(peers));
    }
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < PB_RAY_KEYS; i += blockDim.x)
        if (s_hist[i]) atomicAdd(&hist[i], s_hist[i]);
}
__global__ void __launch_bounds__(1024) k_ray_scan(uint32_t* __restrict__ hist) {  // exclusive prefix sum of the 8192 bins, in place
    __shared__ uint32_t s_part[1024];
    const uint32_t t = threadIdx.x;
    uint32_t v[PB_RAY_KEYS / 1024], sum = 0;
#pragma unroll
    for (int k = 0; k < PB_RAY_KEYS / 1024; ++k) { v[k] = hist[t * (PB_RAY_KEYS / 1024) + k]; sum += v[k]; }
    s_part[t] = sum;
    __syncthreads();
    for (uint32_t off = 1; off < 1024; off <<= 1) {
        uint32_t add = t >= off ? s_part[t - off] : 0;
        __syncthreads();
        s_part[t] += add;
        __syncthreads();
    }
    uint32_t base = s_part[t] - sum;
#pragma unroll
    for (int k = 0; k < PB_RAY_KEYS / 1024; ++k) { hist[t * (PB_RAY_KEYS / 1024) + k] = base; base += v[k]; }
}
__global__ void __launch_bounds__(256) k_ray_scatter(const uint32_t* __restrict__ d_nrays, const uint32_t* __restrict__ keys, uint32_t* __restrict__ cursor,
                                                     uint32_t* __restrict__ perm) {
    const uint32_t n = *d_nrays;
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t total = (n + 31u) & ~31u;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const uint32_t k = i < n ? keys[i] : 0xffffffffu;
        const unsigned peers = __match_any_sync(0xffffffffu, k);
        const int leader = __ffs(peers) - 1;
        uint32_t base = 0;
        if (k != 0xffffffffu && (int)lane == leader) base = atomicAdd(&cursor[k], (uint32_t)__popc(peers));
        base = __shfl_sync(0xffffffffu, base, leader);
        if (k != 0xffffffffu) perm[base + (uint32_t)__popc(peers & ((1u << lane) - 1u))] = i;
    }
}

// Two-level variant of k_ray_scatter (PB_RAY_SORT=2).  The one above issues one global atomicAdd per warp and distinct key;
// on Cornell most of the rays of an iteration hit a handful of hot bins and serialise in L2 (DESIGN.md section 9).  Here every
// CTA owns a contiguous chunk of the queue: it counts the chunk's keys in shared memory, reserves ONE range per (CTA, key) in the
// global cursors, and ranks its rays inside shared memory.  Parity-tested through tests/emu (both modes).
__global__ void __launch_bounds__(256) k_ray_scatter2(const uint32_t* __restrict__ d_nrays, const uint32_t* __restrict__ keys, uint32_t* __restrict__ cursor,
                                                      uint32_t* __restrict__ perm) {
    __shared__ uint32_t s_pos[PB_RAY_KEYS];
    for (uint32_t i = threadIdx.x; i < PB_RAY_KEYS; i += blockDim.x) s_pos[i] = 0;
    __syncthreads();
    const uint32_t n = *d_nrays;
    const uint32_t lane = threadIdx.x & 31;
    uint32_t chunk = (n + gridDim.x - 1) / gridDim.x;
    chunk = (chunk + 31u) & ~31u;  // whole warps
    const uint32_t lo = min(n, blockIdx.x * chunk), hi = min(n, lo + chunk);
    const uint32_t span = ((hi - lo) + 31u) & ~31u;
    for (uint32_t j = threadIdx.x; j < span; j += blockDim.x) {  // count
        const uint32_t i = lo + j;
        const uint32_t k = i < hi ? keys[i] : 0xffffffffu;
        const unsigned peers = __match_any_sync(0xffffffffu, k);
        if (k != 0xffffffffu && (int)lane == __ffs(peers) - 1) atomicAdd(&s_pos[k], (uint32_t)__popc(peers));
    }
    __syncthreads();
    for (uint32_t t = threadIdx.x; t < PB_RAY_KEYS; t += blockDim.x) {  // one global reservation per key the chunk holds
        const uint32_t c = s_pos[t];
        if (c) s_pos[t] = atomicAdd(&cursor[t], c);
    }
    __syncthreads();
    for (uint32_t j = threadIdx.x; j < span; j += blockDim.x) {  // rank inside the reservation
        const uint32_t i = lo + j;
        const uint32_t k = i < hi ? keys[i] : 0xffffffffu;
        const unsigned peers = __match_any_sync(0xffffffffu, k);
        const int leader = __ffs(peers) - 1;
        uint32_t base = 0;
        if (k != 0xffffffffu && (int)lane == leader) base = atomicAdd(&s_pos[k], (uint32_t)__popc(peers));
        base = __shfl_sync(0xffffffffu, base, leader);
        if (k != 0xffffffffu) perm[base + (uint32_t)__popc(peers & ((1u << lane) - 1u))] = i;
    }
}

// -----------------------------------------------------------------------------------------------
// k_shade: shade one path vertex, a surface hit k_sort filed under a shading class: path.rs:95-279, integrator.rs:359-570 (k_sort
// has already finished the previous vertex's estimate_direct).
// Material::compute_scattering_functions of a material with image textures at one hit (e.g. matte.rs:52-86): the bump map first
// (Material::bump, material.rs:116-219, + set_shading_geometry, interaction.rs:345-370: `is` leaves with the new shading frame), then
// the bound textures, then the lobe list of this hit.  Shared by k_texture and the direct / whitted kernels.
__device__ PB_NOINLINE void material_at_hit(const DScene& sc, Isect& is, const UvDiff& dd, DMaterial& m, bool& bumped, bool allow_multiple_lobes) {
    bumped = false;
    const DMatSrc& src = sc.mat_src[is.material];
    if (src.bump) {  // Material::bump (material.rs:116-219) + set_shading_geometry (interaction.rs:345-370), before the other textures
        const uint32_t bt = src.bump - 1u;
        Isect ev = is;
        float du = 0.5f * (fabsf(dd.dudx) + fabsf(dd.dudy));
        if (du == 0.0f) du = 0.0005f;
        ev.p = is.p + is.sh_dpdu * du;  // read by the non-UV mappings only
        ev.uv = make_float2(is.uv.x + du, is.uv.y + 0.0f);
        const float u_displace = texture_evaluate(sc.textures, bt, sc.ewa_lut, ev, dd).r;
        float dv = 0.5f * (fabsf(dd.dvdx) + fabsf(dd.dvdy));
        if (dv == 0.0f) dv = 0.0005f;
        ev.p = is.p + is.sh_dpdv * dv;
        ev.uv = make_float2(is.uv.x + 0.0f, is.uv.y + dv);
        const float v_displace = texture_evaluate(sc.textures, bt, sc.ewa_lut, ev, dd).r;
        const float displace = texture_evaluate(sc.textures, bt, sc.ewa_lut, is, dd).r;
        const V3 dpdu = is.sh_dpdu + is.ns * ((u_displace - displace) / du) + is.sh_dndu * displace;
        const V3 dpdv = is.sh_dpdv + is.ns * ((v_displace - displace) / dv) + is.sh_dndv * displace;
        V3 ns = norm3(cross3(dpdu, dpdv));
        if (is.shape_flips) ns = -ns;
        ns = faceforward3(ns, is.n);
        is.ns = ns;
        is.sh_dpdu = dpdu;
        is.sh_dpdv = dpdv;
        bumped = true;
    }
    float prm[24];
#pragma unroll
    for (int k = 0; k < 24; ++k) prm[k] = src.params[k];
    float au = src.alpha_u, av = src.alpha_v;
    bool float_textured = false;
    for (int g = 0; g < 8; ++g) {
        const uint32_t t = src.tex[g];
        if (!t) continue;
        const Sp v = texture_evaluate(sc.textures, t - 1u, sc.ewa_lut, is, dd);
        const int o = (int)src.tex_off[g];  // params[] offset of the group; spectrum groups come first (pbrt_gpu.h)
        if (g < (int)src.n_spectrum) { prm[o] = v.r; prm[o + 1] = v.g; prm[o + 2] = v.b; }
        else { prm[o] = v.r; float_textured = true; }  // ImageTexture<Float>: one channel, replicated on upload
    }
    if (float_textured) material_alphas_dev(src.kind, prm, au, av);
    compile_material_core(src.kind, prm, au, av, m, allow_multiple_lobes);
}

// k_texture: Material::compute_scattering_functions for the hits on materials with image textures (e.g. matte.rs:61-69): evaluate
// the bound ImageTextures at the hit -- after SurfaceInteraction::compute_differentials (interaction.rs:371-474) for the camera ray,
// with zero differentials for every later ray of the path (spawn_ray carries none, interaction.rs:493-503) -- and compile the
// material's lobe list for this hit into DPaths.slot_mat[slot], where k_shade picks it up.  Launched between k_sort and k_shade,
// only for scenes that have textures.  `camera_ray`: this is the first iteration of the batch (the rays are the camera rays).
__global__ void __launch_bounds__(128) k_texture(DScene sc, DRender rp, DPaths ps, const uint32_t* __restrict__ queue, const uint32_t* __restrict__ d_count,
                                                 uint32_t camera_ray) {
    const uint32_t count = *d_count;
    for (uint32_t qi = blockIdx.x * blockDim.x + threadIdx.x; qi < count; qi += gridDim.x * blockDim.x) {
        const uint32_t slot = queue[qi];
        if (!(__float_as_uint(ps.L[slot].w) & PF_HAS_RAY)) continue;
        const float4 hit = ps.hit[slot];
        const int prim = __float_as_int(hit.x);
        if (prim < 0) continue;
        const uint32_t inst = sc.n_instances ? ps.hit_inst[slot] : 0xffffffffu;
        const float4 rd4 = ps.ray_d[slot];
        V3 wo_unused;
        const Isect is = hit_interaction(sc, rp.instancing, (uint32_t)prim, hit.y, hit.z, hit.w, inst, mk3(rd4.x, rd4.y, rd4.z), wo_unused);
        if (is.material == 0xffffffffu || !(sc.materials[is.material].cls & PB_MAT_TEXTURED)) continue;
        UvDiff dd;
        dd.dudx = dd.dvdx = dd.dudy = dd.dvdy = 0.0f;
        dd.dpdx = dd.dpdy = mk3(0.0f, 0.0f, 0.0f);
        if (camera_ray) {
            const float4 q0 = ps.ray_diff[3 * (size_t)slot], q1 = ps.ray_diff[3 * (size_t)slot + 1], q2 = ps.ray_diff[3 * (size_t)slot + 2];
            dd = compute_differentials(is, mk3(q0.x, q0.y, q0.z), mk3(q0.w, q1.x, q1.y), mk3(q1.z, q1.w, q2.x), mk3(q2.y, q2.z, q2.w));
        }
        Isect isb = is;
        DMaterial m;
        bool bumped;
        material_at_hit(sc, isb, dd, m, bumped, true);  // PathIntegrator: allow_multiple_lobes (path.rs:108)
        if (bumped) {
            ps.slot_frame[2 * (size_t)slot] = make_float4(isb.ns.x, isb.ns.y, isb.ns.z, 0.0f);
            ps.slot_frame[2 * (size_t)slot + 1] = make_float4(isb.sh_dpdu.x, isb.sh_dpdu.y, isb.sh_dpdu.z, 0.0f);
        }
        ps.slot_mat[slot] = m;
    }
}

// INST: the scene has object instances (hits may need carrying back to world space); compiled out of the variants the
// instance-free scenes run, so that their code is the measured one.
// SPEC = 1 + k: the instantiation for the shading class "a single lobe of kind k" -- untextured matte (Lambert / Oren-Nayar), metal,
// substrate, mirror, smooth glass -- with the BSDF code folded to that one lobe (pb_bsdf.cuh): a fraction of the general kernel's
// instructions.  The host launches one instantiation per class the scene has and
// the general one (SPEC = 0) over the multi-lobe / textured classes that are left; [cls_lo, cls_hi) is the launch's class range.
#ifndef PB_SHADE_SPEC_BLOCKS
// Resident CTAs per SM the specialised instantiation is compiled for (register budget 65536 / (128 * n)).  5 and 6 make ptxas spill
// (104-200 B of stack) and were slower on the statue, Cornell and the conference scene on an H100 SXM (700 W).
#define PB_SHADE_SPEC_BLOCKS 4
#endif
template <int LIGHTS, bool HALTON, bool INST, int SPEC>
__global__ void __launch_bounds__(PB_SHADE_THREADS, (SPEC >= 1 ? PB_SHADE_SPEC_BLOCKS : 4)) k_shade(DScene sc, DRender rp, DPaths ps, DLightGrid grid, const uint32_t* __restrict__ nib,
                                                          uint32_t sobol_cfg, uint32_t n_chunks, const uint32_t* __restrict__ cls_queue,
                                                          uint32_t cls_stride, const uint32_t* __restrict__ cls_count, uint32_t* __restrict__ queue_out,
                                                          uint32_t* __restrict__ d_count_out, float4* __restrict__ rays, uint32_t* __restrict__ d_nrays,
                                                          DCounters* cnt, uint32_t* __restrict__ d_error, uint32_t* __restrict__ ray_keys, uint32_t key_mask,
                                                          uint32_t* __restrict__ reset_cursor, uint32_t* __restrict__ reset_requests,
                                                          uint32_t* __restrict__ reset_cls_count, uint32_t cls_lo, uint32_t cls_hi) {
    PB_DYNAMIC_SMEM(smem_raw);
    __shared__ __align__(8) uint64_t s_bar;
    if (blockIdx.x == 0 && threadIdx.x < PB_SHADE_CLASSES) {  // see k_sort
        reset_cls_count[threadIdx.x] = 0u;
        if (threadIdx.x == 0) { *reset_cursor = 0u; if (reset_requests) *reset_requests = 0u; }
    }
    // Sobol' nibble tables of the dimensions / index bits this render can reach: TMA bulk copies -> shared memory
    const uint32_t* tab = nib;
    // `nib` is this render's transposed slice nibT[(chunk*16+e)*ds + dim] with ds = sobol_cfg & 0xffff; bit 31 = stage it in shared memory
    const uint32_t tab_stride = sobol_cfg & 0xffffu;
    if (!HALTON && (sobol_cfg >> 31)) {
        const uint32_t bytes = n_chunks * 64u * tab_stride;
        if (threadIdx.x == 0) {
            mbar_init(&s_bar, 1);
            mbar_fence_init();
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            mbar_expect_tx(&s_bar, bytes);
            for (uint32_t off = 0; off < bytes; off += 16384u)  // one bulk copy per 16 KB
                tma_bulk_g2s(smem_raw + off, reinterpret_cast<const unsigned char*>(nib) + off, min(16384u, bytes - off), &s_bar);
        }
        mbar_wait(&s_bar, 0);
        tab = reinterpret_cast<const uint32_t*>(smem_raw);
    }
    __shared__ uint32_t s_tiles[PB_SHADE_CLASSES + 1];  // exclusive prefix of 32-slot tiles per class
    if (threadIdx.x == 0) {
        uint32_t acc = 0;
        for (uint32_t c = 0; c < PB_SHADE_CLASSES; ++c) { s_tiles[c] = acc; if (c >= cls_lo && c < cls_hi) acc += (cls_count[c] + 31u) >> 5; }
        s_tiles[PB_SHADE_CLASSES] = acc;
    }
    __syncthreads();
    const uint32_t total_tiles = s_tiles[PB_SHADE_CLASSES];
    const int NONSPEC = BSDF_ALL & ~BSDF_SPECULAR;
    const float inf = __int_as_float(0x7f800000);
    uint32_t n_light_tests = 0, n_slots = 0, n_vertices = 0;
    const uint32_t warps_total = (gridDim.x * blockDim.x) >> 5;
    const uint32_t warp_id = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31;
    for (uint32_t tile = warp_id; tile < total_tiles; tile += warps_total) {
        // every warp handles 32 slots of ONE class: warps never mix two lobe sets
        uint32_t cls = 0;
        while (cls + 1 < PB_SHADE_CLASSES && tile >= s_tiles[cls + 1]) ++cls;
        const uint32_t qi = (tile - s_tiles[cls]) * 32u + lane;
        const uint32_t count = cls_count[cls];
        bool push = false, emit_ext = false, emit_sh = false, emit_mis = false;
        float4 ext0, ext1, sh0, sh1, mis0, mis1;
        ext0 = ext1 = sh0 = sh1 = mis0 = mis1 = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        uint32_t slot = 0;
        if (qi < count) {
            slot = cls_queue[(size_t)cls * cls_stride + qi];
            n_slots++;
            // all per-slot state is fetched up front so that the loads overlap (the kernel is latency bound)
            const float4 Lf = ps.L[slot];
            const float4 st_hit = ps.hit[slot], st_rd = ps.ray_d[slot], st_beta = ps.beta[slot];
            const uint2 st_sobol = ps.sobol[slot];
            const uint32_t st_dim = ps.dim[slot];
            uint32_t flags = __float_as_uint(Lf.w);
            Sp L = mksp(Lf.x, Lf.y, Lf.z);
            uint32_t out_flags = 0;  // terminated unless set below
            uint32_t bounces = flags >> PF_BOUNCES_SHIFT;
            bool specular_bounce = (flags & PF_SPECULAR_BOUNCE) != 0;
            const float4 hit = st_hit;
            int prim = __float_as_int(hit.x);  // k_sort files surface hits only: PF_HAS_RAY is set and prim >= 0
            n_vertices++;
            const float4 rd4 = st_rd, b4 = st_beta;
            V3 rd = mk3(rd4.x, rd4.y, rd4.z);
            Sp beta = mksp(b4.x, b4.y, b4.z);
            float eta_scale = b4.w;
            V3 wo = -rd;
            V3 wo_nee = wo;  // isect.wo: what estimate_direct evaluates the BSDF with (differs for a transformed instance hit)
            Isect is = INST ? hit_interaction(sc, rp.instancing, (uint32_t)prim, hit.y, hit.z, hit.w, ps.hit_inst[slot], rd, wo_nee)
                                      : tri_interaction(sc, (uint32_t)prim, hit.y, hit.z, hit.w);
            if (bounces == 0 || specular_bounce) {
                // `l += beta * isect.le(&-ray.d)` (path.rs:97-100) also for a surface that emits nothing: le() is then black (interaction.rs:475-483),
                // and beta * 0 is NaN when a degenerate BSDF value has made a component of beta infinite.  (The reference asserts on an infinite
                // beta.y() right after the update, path.rs:158-171, so it aborts before it gets here; the oracle restates the arithmetic without
                // the asserts, and this statement keeps the two restatements equal there too: the sample ends as NaN and k_resolve's has_nans()
                // drops it -- tests/test_emu_kernels.py::test_randomised_materials_and_settings.)
                const Sp le = is.area_light >= 0 ? light_L(sc.lights[is.area_light], is.n, wo) : sp1(0.0f);
                L = L + beta * le;
            }
            if (bounces < rp.max_depth) {
                if (is.material == 0xffffffffu) {  // null BSDF: pass through, bounce not counted (path.rs:109-116)
                    V3 o = offset_ray_origin(is.p, is.p_error, is.n, rd);
                    ext0 = make_float4(o.x, o.y, o.z, inf);
                    ext1 = make_float4(rd.x, rd.y, rd.z, __uint_as_float(slot | (RAY_EXTEND << 30)));
                    emit_ext = true;
                    out_flags = (flags & ~0xffu) | (flags & PF_SPECULAR_BOUNCE) | PF_HAS_RAY;
                } else {
                    BsdfFrame B;
                    B.mat = sc.materials + is.material;
                    if (SPEC == 0 && (B.mat->cls & PB_MAT_TEXTURED)) {
                        if (B.mat->cls & PB_MAT_BUMPED) {  // the bump-mapped shading frame of this hit (k_texture)
                            const float4 f0 = ps.slot_frame[2 * (size_t)slot], f1 = ps.slot_frame[2 * (size_t)slot + 1];
                            is.ns = mk3(f0.x, f0.y, f0.z);
                            is.sh_dpdu = mk3(f1.x, f1.y, f1.z);  // the frame below is built from these two
                        }
                        B.mat = ps.slot_mat + slot;  // lobes of this hit, compiled by k_texture
                    }
                    B.ns = is.ns;
                    B.ng = is.n;
                    B.ss = norm3(is.sh_dpdu);
                    B.ts = cross3(is.ns, B.ss);
                    const uint2 si = st_sobol;
                    SobolT sob;
                    sob.nib = tab;
                    sob.ds = tab_stride;
                    sob.n_chunks = n_chunks;
                    sob.index = ((uint64_t)si.y << 32) | si.x;
                    sob.dim = st_dim;
                    sob.overflow = false;
                    uint32_t nee_flags = 0;
                    if (SPEC >= 1 ? pb_spec_has_nonspecular(SPEC) : (B.mat->nonspecular > 0)) {
                        // uniform_sample_one_light (integrator.rs:359-403); its result is added as
                        // L += beta * Ld right here unless rays have to be traced first
                        Sp ld_now = sp1(0.0f);
                        const int nl = grid.n_lights;
                        if (nl > 0) {
                            const size_t v = (rp.light_strategy == 2u) ? grid.row_of(light_voxel(sc, grid, is.p)) : (size_t)0;
                            float choice_pdf;
                            // light choice, u_light, u_scattering: five consecutive dimensions in one pass
                            float u5[5];
                            if (HALTON) {
#pragma unroll
                                for (int k = 0; k < 5; ++k) u5[k] = halton_scrambled(rp, (uint32_t)sob.index, min(sob.dim + (uint32_t)k, (uint32_t)(PB_HALTON_DIMS - 1)));
                            } else sobolT_fill<5>(sob, u5);
                            const float u_choice = sobolT_take<HALTON>(sob, 1) ? u5[0] : 0.0f;
                            int light_num = sample_discrete(grid.func + v * nl, grid.cdf + v * (nl + 1), grid.func_int[v], nl,
                                                            u_choice, choice_pdf);
                            if (choice_pdf != 0.0f) {
                                float2 u_light = make_float2(0.0f, 0.0f), u_scat = make_float2(0.0f, 0.0f);
                                if (sobolT_take<HALTON>(sob, 2)) u_light = make_float2(u5[1], u5[2]);
                                if (sobolT_take<HALTON>(sob, 2)) u_scat = make_float2(u5[3], u5[4]);
                                const DLight& light = sc.lights[light_num];
                                // estimate_direct (integrator.rs:406-570): light-sampling strategy
                                V3 wi = mk3(0.0f, 0.0f, 0.0f);
                                float light_pdf = 0.0f, scattering_pdf = 0.0f, mis_w = 0.0f;
                                Sp a = sp1(0.0f);
                                LightSample ls;
                                Sp li = light_sample_li<LIGHTS>(sc, light, is.p, u_light, wi, light_pdf, ls);
                                if (light_pdf > 0.0f && !is_black(li)) {
                                    Sp f = bsdf_f<SPEC>(B, wo_nee, wi, NONSPEC) * sp1(absdot3(wi, is.ns));
                                    scattering_pdf = bsdf_pdf<SPEC>(B, wo_nee, wi, NONSPEC);
                                    if (!is_black(f)) {
                                        // VisibilityTester::unoccluded -> spawn_ray_to (interaction.rs:81-94)
                                        V3 origin = offset_ray_origin(is.p, is.p_error, is.n, ls.p - is.p);
                                        V3 target = offset_ray_origin(ls.p, ls.p_error, ls.n, origin - ls.p);
                                        V3 sd = target - origin;
                                        if (LIGHTS != 0 && light_is_delta<LIGHTS>(light)) a = f * li / light_pdf;  // is_delta_light: no MIS
                                        else {
                                            float w = power_heuristic(light_pdf, scattering_pdf);
                                            a = f * li * sp1(w) / light_pdf;
                                        }
                                        sh0 = make_float4(origin.x, origin.y, origin.z, 1.0f - PB_SHADOW_EPSILON);
                                        sh1 = make_float4(sd.x, sd.y, sd.z, __uint_as_float(slot | (RAY_SHADOW << 30)));
                                        emit_sh = true;
                                        nee_flags |= PF_HAS_SHADOW;
                                    }
                                }
                                // BSDF-sampling strategy (skipped for delta lights, integrator.rs:480); `wi` is shared
                                // with the light strategy as in the reference, sampled_type = 0 in (quirk Q8)
                                int st = 0;
                                Sp f2 = sp1(0.0f);
                                if (LIGHTS == 0 || !light_is_delta<LIGHTS>(light)) {
                                    f2 = bsdf_sample_f<SPEC>(B, wo_nee, wi, u_scat, scattering_pdf, NONSPEC, st);
                                    f2 = f2 * sp1(absdot3(wi, is.ns));
                                }
                                if (!is_black(f2) && scattering_pdf > 0.0f) {
                                    V3 mo = offset_ray_origin(is.p, is.p_error, is.n, wi);  // it.spawn_ray(wi)
                                    if (LIGHTS == 0 || light.kind == 0u) n_light_tests++;  // Triangle::intersect inside pdf_li (area lights only)
                                    float lp = light_pdf_li<LIGHTS>(sc, light, is.p, mo, wi);
                                    if (lp != 0.0f) {
                                        mis_w = power_heuristic(scattering_pdf, lp);
                                        mis0 = make_float4(mo.x, mo.y, mo.z, inf);
                                        mis1 = make_float4(wi.x, wi.y, wi.z, __uint_as_float(slot | (RAY_MIS << 30)));
                                        emit_mis = true;
                                        ps.mis_d[slot] = make_float4(wi.x, wi.y, wi.z, __uint_as_float((uint32_t)light_num));
                                        ps.mis_f[slot] = make_float4(f2.r, f2.g, f2.b, scattering_pdf);
                                        nee_flags |= PF_HAS_MIS;
                                    }
                                }
                                if (nee_flags) {
                                    ps.ld_light[slot] = make_float4(a.r, a.g, a.b, mis_w);
                                    ps.nee_beta[slot] = make_float4(beta.r, beta.g, beta.b, choice_pdf);
                                } else ld_now = spdiv0(sp1(0.0f), choice_pdf);
                            }
                        }
                        if (!nee_flags) L = L + beta * ld_now;
                    }
                    // sample the BSDF for the next direction (path.rs:141-188)
                    V3 wi = mk3(0.0f, 0.0f, 0.0f);
                    float pdf = 0.0f;
                    int st = 255;
                    float u3[3];  // BSDF sample + the Russian-roulette dimension behind it
                    if (HALTON) {
                        u3[0] = halton_scrambled(rp, (uint32_t)sob.index, min(sob.dim, (uint32_t)(PB_HALTON_DIMS - 1)));
                        u3[1] = halton_scrambled(rp, (uint32_t)sob.index, min(sob.dim + 1u, (uint32_t)(PB_HALTON_DIMS - 1)));
                        u3[2] = 0.0f;  // the roulette dimension is drawn only when it is needed (below)
                    } else sobolT_fill<3>(sob, u3);
                    const float2 u_bsdf = sobolT_take<HALTON>(sob, 2) ? make_float2(u3[0], u3[1]) : make_float2(0.0f, 0.0f);
                    Sp f = bsdf_sample_f<SPEC>(B, wo, wi, u_bsdf, pdf, BSDF_ALL, st);
                    bool alive = !(is_black(f) || pdf == 0.0f);
                    if (alive) {
                        beta = beta * ((f * absdot3(wi, is.ns)) / pdf);
                        specular_bounce = (st & BSDF_SPECULAR) != 0;
                        if ((st & BSDF_SPECULAR) && (st & BSDF_TRANSMISSION)) {
                            float eta = B.mat->eta;
                            if (dot3(wo, is.n) > 0.0f) eta_scale *= eta * eta;
                            else eta_scale *= 1.0f / (eta * eta);
                        }
                        V3 o = offset_ray_origin(is.p, is.p_error, is.n, wi);
                        // Russian roulette (path.rs:251-262)
                        Sp rr_beta = beta * eta_scale;
                        if (maxsp(rr_beta) < rp.rr_threshold && bounces > 3) {
                            float q = fmaxf(0.05f, 1.0f - maxsp(rr_beta));
                            if (HALTON) u3[2] = halton_scrambled(rp, (uint32_t)sob.index, min(sob.dim, (uint32_t)(PB_HALTON_DIMS - 1)));
                            const float u_rr = sobolT_take<HALTON>(sob, 1) ? u3[2] : 0.0f;
                            if (u_rr < q) alive = false;
                            else beta = beta / (1.0f - q);
                        }
                        if (alive) {
                            ext0 = make_float4(o.x, o.y, o.z, inf);
                            ext1 = make_float4(wi.x, wi.y, wi.z, __uint_as_float(slot | (RAY_EXTEND << 30)));
                            emit_ext = true;
                            ps.ray_d[slot] = make_float4(wi.x, wi.y, wi.z, 0.0f);
                            ps.beta[slot] = make_float4(beta.r, beta.g, beta.b, eta_scale);
                            ps.dim[slot] = sob.dim;
                            out_flags = ((bounces + 1) << PF_BOUNCES_SHIFT) | (specular_bounce ? PF_SPECULAR_BOUNCE : 0u) | PF_HAS_RAY;
                        }
                    }
                    out_flags |= nee_flags;
                    if (sob.overflow) atomicOr(d_error, 1u);
                }
            }
            ps.L[slot] = make_float4(L.r, L.g, L.b, __uint_as_float(out_flags));
            push = (out_flags & (PF_HAS_RAY | PF_HAS_SHADOW | PF_HAS_MIS)) != 0;
        }
        // ---- compaction: survivors -> next shade queue, their rays -> ray queue (warp ballot + prefix sum,
        // one atomic per queue and warp)
        const unsigned mp = __ballot_sync(0xffffffffu, push);
        const unsigned me = __ballot_sync(0xffffffffu, emit_ext), mm = __ballot_sync(0xffffffffu, emit_mis), ms = __ballot_sync(0xffffffffu, emit_sh);
        const uint32_t ne = (uint32_t)__popc(me), nm = (uint32_t)__popc(mm), nsh = (uint32_t)__popc(ms);
        uint32_t qbase = 0, rbase = 0;
        if (lane == 0) {  // both atomics are in flight together
            if (mp) qbase = atomicAdd(d_count_out, (uint32_t)__popc(mp));
            if (ne + nm + nsh) rbase = atomicAdd(d_nrays, ne + nm + nsh);
        }
        qbase = __shfl_sync(0xffffffffu, qbase, 0);
        rbase = __shfl_sync(0xffffffffu, rbase, 0);
        if (push) queue_out[qbase + (uint32_t)__popc(mp & ((1u << lane) - 1u))] = slot;
        const unsigned lt = (1u << lane) - 1u;
        if (emit_ext) { size_t q = rbase + (uint32_t)__popc(me & lt); rays[2 * q] = ext0; rays[2 * q + 1] = ext1; if (ray_keys) ray_keys[q] = ray_key(sc, ext0, ext1) & key_mask; }
        if (emit_mis) { size_t q = rbase + ne + (uint32_t)__popc(mm & lt); rays[2 * q] = mis0; rays[2 * q + 1] = mis1; if (ray_keys) ray_keys[q] = ray_key(sc, mis0, mis1) & key_mask; }
        if (emit_sh) { size_t q = rbase + ne + nm + (uint32_t)__popc(ms & lt); rays[2 * q] = sh0; rays[2 * q + 1] = sh1; if (ray_keys) ray_keys[q] = ray_key(sc, sh0, sh1) & key_mask; }
    }
    uint32_t t = warp_sum(n_light_tests);
    if (lane == 0 && t) atomicAdd(&cnt->light_tri_tests, (unsigned long long)t);
    t = warp_sum(n_slots);
    if (lane == 0 && t) atomicAdd(&cnt->shade_slots, (unsigned long long)t);
    t = warp_sum(n_vertices);
    if (lane == 0 && t) atomicAdd(&cnt->shaded_vertices, (unsigned long long)t);
}

// -----------------------------------------------------------------------------------------------
// AOIntegrator (src/integrators/ao.rs:47-97) on the same ray-generation, trace and film kernels.  A camera sample s of a pixel
// takes ao_n directions from the sampler's 2D sample array: entry s*ao_n + k of that array is dimensions 5 / 6 of the pixel's
// sample number s*ao_n + k (GlobalSampler::start_pixel, sobol.rs:165-177 / halton.rs:286-298).  k_ao_shade: one thread per
// (camera sample, k) rebuilds the hit's frame, draws the direction and writes an any-hit ray plus its weight dot(wi,n)/(pdf n);
// k_trace fills the occlusion flags; k_ao_resolve adds the weights of the unoccluded directions in k order.
// GPU parity: tests/test_gpu_parity_siblings.py.
PB_D V3 uniform_sample_hemisphere(float2 u) {  // sampling.rs:309-318
    float z = u.x;
    float r = sqrtf(fmaxf(0.0f, 1.0f - z * z));
    float phi = 2.0f * PB_PI * u.y;
    float sp, cp;
    sincos_rn(phi, sp, cp);
    return mk3(r * cp, r * sp, z);
}
__global__ void __launch_bounds__(256) k_ao_shade(DScene sc, DRender rp, DPaths ps, BatchInfo bi, uint32_t ao_n, uint32_t ao_cos, const uint32_t* __restrict__ nib,
                                                  uint32_t n_chunks, const uint64_t* __restrict__ vdc, const uint64_t* __restrict__ vdci,
                                                  float4* __restrict__ rays, float* __restrict__ weight, uint32_t* __restrict__ d_nrays) {
    __shared__ uint64_t s_vdc[52], s_vdci[52];
    if (threadIdx.x < 52) {
        uint32_t m = rp.log2_res;
        s_vdc[threadIdx.x] = m ? vdc[(m - 1) * 52 + threadIdx.x] : 0;
        s_vdci[threadIdx.x] = m ? vdci[(m - 1) * 52 + threadIdx.x] : 0;
    }
    __syncthreads();
    const uint32_t n_paths = bi.n_pixels * bi.n_samples;
    const uint64_t total = (uint64_t)n_paths * ao_n;
    const uint64_t gid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;  // (camera sample, k); the host keeps total < 2^30
    float4 r0 = make_float4(0.0f, 0.0f, 0.0f, 0.0f), r1 = r0;
    bool live = false;
    if (gid < total) {
        const uint32_t slot = (uint32_t)(gid / ao_n), k = (uint32_t)(gid % ao_n);
        float w = __int_as_float(0x7fc00000);  // NaN: no direction drawn, nothing to add
        const uint32_t flags = __float_as_uint(ps.L[slot].w);
        const float4 hit = ps.hit[slot];
        const int prim = __float_as_int(hit.x);
        if ((flags & PF_HAS_RAY) && prim >= 0) {
            const float4 rd4 = ps.ray_d[slot];
            const V3 rd = mk3(rd4.x, rd4.y, rd4.z);
            V3 wo_unused;
            const Isect is = sc.n_instances ? hit_interaction(sc, rp.instancing, (uint32_t)prim, hit.y, hit.z, hit.w, ps.hit_inst[slot], rd, wo_unused)
                                            : tri_interaction(sc, (uint32_t)prim, hit.y, hit.z, hit.w);
            const V3 n = faceforward3(is.n, -rd);
            const V3 s = norm3(is.dpdu);
            const V3 t = cross3(is.n, s);
            // the array entry: pixel sample number s_pix * ao_n + k, dimensions 5 (x) and 6 (y)
            const uint32_t pl = slot / bi.n_samples, s_pix = bi.first_sample + slot % bi.n_samples;
            const uint32_t pix = bi.first_pixel + pl;
            int px, py;
            share_pixel(rp, pix, px, py);
            const uint64_t j = (uint64_t)s_pix * ao_n + k;
            float2 u;
            if (rp.halton) {
                const uint64_t index = halton_index(rp, px, py, j);
                u = make_float2(halton_sample_dimension(rp, index, 5u), halton_sample_dimension(rp, index, 6u));
            } else {
                SobolCtx sob;
                sob.nib = nib; sob.stride = PB_SOBOL_CHUNKS; sob.n_chunks = n_chunks; sob.dim = 0; sob.overflow = false;
                sob.index = sobol_interval_to_index(s_vdc, s_vdci, rp.log2_res, j, px - rp.sb[0], py - rp.sb[1]);
                u = make_float2(sobol_sample_nib(sob, 5), sobol_sample_nib(sob, 6));
            }
            V3 wl;
            float pdf;
            if (ao_cos) { wl = cosine_sample_hemisphere(u); pdf = fabsf(wl.z) * PB_INV_PI; }
            else { wl = uniform_sample_hemisphere(u); pdf = PB_INV_2_PI; }
            const V3 wi = mk3(s.x * wl.x + t.x * wl.y + n.x * wl.z, s.y * wl.x + t.y * wl.y + n.y * wl.z, s.z * wl.x + t.z * wl.y + n.z * wl.z);
            if (pdf != 0.0f) {
                const V3 o = offset_ray_origin(is.p, is.p_error, is.n, wi);  // isect.spawn_ray(wi)
                r0 = make_float4(o.x, o.y, o.z, __int_as_float(0x7f800000));
                r1 = make_float4(wi.x, wi.y, wi.z, __uint_as_float((uint32_t)gid | (RAY_SHADOW << 30)));
                w = dot3(wi, n) / (pdf * (float)ao_n);
                live = true;
            }
        }
        weight[gid] = w;
    }
    const uint32_t pos = queue_append(d_nrays, live);  // *d_nrays is zeroed by the host before the launch
    if (live) { rays[2 * (size_t)pos] = r0; rays[2 * (size_t)pos + 1] = r1; }
}
__global__ void __launch_bounds__(256) k_ao_resolve(DPaths ps, BatchInfo bi, uint32_t ao_n, const float* __restrict__ weight, const uint32_t* __restrict__ occl) {
    const uint32_t n_paths = bi.n_pixels * bi.n_samples;
    const uint32_t slot = blockIdx.x * blockDim.x + threadIdx.x;
    if (slot >= n_paths) return;
    float l = 0.0f;
    for (uint32_t k = 0; k < ao_n; ++k) {  // the reference's order: l += Spectrum(w_k) for k = 0, 1, ...
        const float w = weight[(size_t)slot * ao_n + k];
        if (w == w && occl[(size_t)slot * ao_n + k] == 0u) l += w;
    }
    const float4 L = ps.L[slot];
    ps.L[slot] = make_float4(l, l, l, L.w);
}

// The single reduce of the multi-device render (pbrt_gpu_render_multi; SURVEY.md 8e): dst[i] += sum_k src[k][i] over the films of
// the peer devices, read straight out of their memory through NVLink / NVSwitch peer access by the device that owns dst.
struct PeerFilms { const float4* p[15]; int n; };
__global__ void __launch_bounds__(256) k_film_sum_peers(float4* __restrict__ dst, PeerFilms peers, size_t n4) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
        float4 a = dst[i];
        for (int k = 0; k < peers.n; ++k) {
            const float4 b = peers.p[k][i];
            a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
        }
        dst[i] = a;
    }
}

// known-answer hook for AnimatedTransform::interpolate (pbrt_gpu_kat_animated_interpolate)
__global__ void k_kat_motion(const DMotion mo, const float* __restrict__ t, uint32_t n, float* __restrict__ m, float* __restrict__ m_inv) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) motion_interpolate(mo, t[i], m + 16 * (size_t)i, m_inv + 16 * (size_t)i);
}
// known-answer hook for the realistic camera's generate_ray_differential (pbrt_gpu_kat_realistic_rays): in[i] = {p_film, p_lens},
// time[i]; out: 19 floats per sample, o[3] d[3] weight rx_o[3] ry_o[3] rx_d[3] ry_d[3], zeros where the weight is 0
__global__ void k_kat_realistic(const DScene sc, const DLens lens, const DMotion cam_mo, uint32_t cam_motion, const float4* __restrict__ in,
                                const float* __restrict__ time, uint32_t n, float* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float c2w_t[16], c2w_inv_t[16];
    if (cam_motion) motion_interpolate(cam_mo, lerpf(time[i], sc.shutter_open, sc.shutter_close), c2w_t, c2w_inv_t);
    const float4 q = in[i];
    V3 o, d, rxo, ryo, rxd, ryd;
    const float wt = lens_generate_ray_differential(lens, cam_motion ? c2w_t : sc.camera_to_world, make_float2(sc.shutter_open, sc.shutter_close),
                                                    make_float2(q.x, q.y), make_float2(q.z, q.w), o, d, rxo, ryo, rxd, ryd);
    float* r = out + 19 * (size_t)i;
    const V3 v[6] = {o, d, rxo, ryo, rxd, ryd};
    for (int k = 0; k < 6; ++k) {
        r[(k < 2 ? 3 * k : 3 * k + 1)] = wt != 0.0f ? v[k].x : 0.0f;
        r[(k < 2 ? 3 * k : 3 * k + 1) + 1] = wt != 0.0f ? v[k].y : 0.0f;
        r[(k < 2 ? 3 * k : 3 * k + 1) + 2] = wt != 0.0f ? v[k].z : 0.0f;
    }
    r[6] = wt;
}
// known-answer hook for the device sin/cos (pbrt_gpu_kat_sincos)
__global__ void k_kat_sincos(const float* __restrict__ x, uint32_t n, float* __restrict__ s, float* __restrict__ c) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float a, b;
    sincos_rn(x[i], a, b);
    // the separate entry points must agree with the fused one
    if (__float_as_uint(sin_rn(x[i])) != __float_as_uint(a) || __float_as_uint(cos_rn(x[i])) != __float_as_uint(b)) a = b = __int_as_float(0x7fc00000);
    s[i] = a; c[i] = b;
}
__global__ void k_kat_log2(const float* __restrict__ x, uint32_t n, float* __restrict__ y) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) y[i] = log2_rn(x[i]);
}
__global__ void k_kat_acos_atan2(const float* __restrict__ x, const float* __restrict__ y, uint32_t n, float* __restrict__ ac, float* __restrict__ at) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    ac[i] = acos_rn(x[i]);
    at[i] = atan2_rn(y[i], x[i]);
}

// -----------------------------------------------------------------------------------------------
// k_resolve: FilmTile::add_sample (film.rs:94-147) for every sample of a pixel, in sample order.
// Contributions to the sample's own pixel are summed in registers in the reference's order; the
// rare contributions to neighbouring pixels (filter footprint, sobol.rs:132-137 apron case) use
// atomics, like the unordered tile merge of the reference (integrator.rs:209-215).
// WEIGHTED: the realistic camera's ray weights (k_raygen's DLens.weight), multiplied in the reference's order L * weight * filter
// weight; every other camera's weight is 1 and its instantiation never reads `weight`.
template <bool WEIGHTED>
__global__ void __launch_bounds__(256) k_resolve(DRender rp, DPaths ps, BatchInfo bi, const float* __restrict__ filter_table, float* __restrict__ film,
                                                float* __restrict__ sample_rgb, const float* __restrict__ weight) {
    uint32_t pl = blockIdx.x * blockDim.x + threadIdx.x;
    if (pl >= bi.n_pixels) return;
    uint32_t pix = bi.first_pixel + pl;
    int px, py;
    if (!share_pixel(rp, pix, px, py)) return;  // the part of an edge tile beyond the sample bounds: no samples were drawn
    const int fw = rp.cb[2] - rp.cb[0];
    float ar = 0.0f, ag = 0.0f, ab = 0.0f, aw = 0.0f;
    bool own_inside = px >= rp.cb[0] && px < rp.cb[2] && py >= rp.cb[1] && py < rp.cb[3];
    const float inv_rx = 1.0f / rp.filter_radius[0], inv_ry = 1.0f / rp.filter_radius[1];
    for (uint32_t s = 0; s < bi.n_samples; ++s) {
        uint32_t slot = pl * bi.n_samples + s;
        float2 pf = ps.p_film[slot];
        if (pf.x != pf.x) continue;  // pixel outside the integrator's pixel bounds
        float4 Lf = ps.L[slot];
        Sp l = mksp(Lf.x, Lf.y, Lf.z);
        if (has_nans(l)) l = sp1(0.0f);  // integrator.rs:165-173 (the other two checks can never fire, quirk Q1)
        if (sample_rgb) {
            float* o = sample_rgb + ((size_t)pix * rp.spp + bi.first_sample + s) * 3;
            o[0] = l.r; o[1] = l.g; o[2] = l.b;
        }
        if (lum(l) > rp.max_sample_luminance) l = l * sp1(rp.max_sample_luminance / lum(l));
        float dx = pf.x - 0.5f, dy = pf.y - 0.5f;
        int p0x = max(f2i_sat(ceilf(dx - rp.filter_radius[0])), rp.cb[0]), p0y = max(f2i_sat(ceilf(dy - rp.filter_radius[1])), rp.cb[1]);
        int p1x = min(f2i_sat(floorf(dx + rp.filter_radius[0])) + 1, rp.cb[2]), p1y = min(f2i_sat(floorf(dy + rp.filter_radius[1])) + 1, rp.cb[3]);
        for (int y = p0y; y < p1y; ++y) {
            float fy = fabsf(((float)y - dy) * inv_ry * 16.0f);
            int iy = f2i_sat(fminf(floorf(fy), 15.0f));
            for (int x = p0x; x < p1x; ++x) {
                float fx = fabsf(((float)x - dx) * inv_rx * 16.0f);
                int ix = f2i_sat(fminf(floorf(fx), 15.0f));
                float w = __ldg(filter_table + iy * 16 + ix);
                Sp c = l * sp1(WEIGHTED ? weight[slot] : 1.0f) * sp1(w);  // sample_weight = 1 but for the realistic camera
                if (x == px && y == py) { ar += c.r; ag += c.g; ab += c.b; aw += w; }
                else {
                    float* d = film + 4 * ((size_t)(y - rp.cb[1]) * fw + (x - rp.cb[0]));
                    atomicAdd(d, c.r); atomicAdd(d + 1, c.g); atomicAdd(d + 2, c.b); atomicAdd(d + 3, w);
                }
            }
        }
    }
    if (own_inside) {
        float* d = film + 4 * ((size_t)(py - rp.cb[1]) * fw + (px - rp.cb[0]));
        atomicAdd(d, ar); atomicAdd(d + 1, ag); atomicAdd(d + 2, ab); atomicAdd(d + 3, aw);
    }
}

}  // namespace pb
