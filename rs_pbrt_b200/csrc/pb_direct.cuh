// pb_direct.cuh -- DirectLightingIntegrator (src/integrators/directlighting.rs:70-260) and WhittedIntegrator
// (src/integrators/whitted.rs:43-254) as a wavefront.
//
// Both integrators are a recursion: L(node) = Le + direct light + f_r * L(reflected child) * |cos|/pdf + f_t * L(transmitted child)
// * |cos|/pdf, both children while depth + 1 < max_depth.  Float addition is not associative and the sampler's dimensions are
// handed out in call order, so the tree is walked depth first, exactly in the reference's order, by a small state machine per
// camera sample: a stack of partial sums (node_L), the multiplier that a node's result gets in its parent (node_mul), and what is
// needed to come back to a node for its transmission ray after the reflected subtree has returned (its hit record and incoming
// direction).  Per iteration: k_trace -> k_direct_step (one thread per camera sample: fold the direct light that was pending, take
// the traced ray's hit, return through finished nodes, emit at most one new ray) -> k_direct_nee (one thread per (camera sample,
// light sample): estimate_direct's shadow and MIS rays for the node shaded in this iteration) -> k_trace ...
#pragma once
#include "pb_kernels.cuh"

namespace pb {

#define PB_DIRECT_MAX_DEPTH 8
enum { DS_DONE = 0u, DS_WAIT_TRACE = 1u, DS_COMPLETE_PENDING = 2u };
enum { STAGE_NONE = 0u, STAGE_AFTER_REFLECT = 1u, STAGE_AFTER_TRANSMIT = 2u };

struct DDirect {
    uint32_t max_depth;
    uint32_t n_nee;        // light samples per node: "all" sum of n_samples, "one" 1, whitted n_lights
    uint32_t whitted, sample_all;
    uint32_t n_arrays;     // 2D sample arrays requested by preprocess: 2 * n_lights * max_depth ("all"), else 0
    uint32_t array_end;    // first regular dimension: 5 + 2 * n_arrays (GlobalSampler)
    uint32_t n_chunks;     // Sobol' index chunks covering the array sample numbers
    const uint32_t* nee_light;  // [n_nee] light of light sample q
    const uint32_t* nee_k;      // [n_nee] its k within that light
    const uint32_t* light_n;    // [n_lights] n_samples of each light
    const uint32_t* light_q0;   // [n_lights] first q of each light
    size_t cap;
    // per slot
    uint32_t* state;
    int* depth;
    uint32_t* arr_off;     // array_2d_offset of the sampler
    int* nee_depth;        // node whose direct light is in flight (-1: none)
    uint32_t* nee_dim;     // sampler state at that node's light loop
    uint32_t* nee_arr;
    uint32_t* fresh;       // the node was shaded in this iteration: k_direct_nee has work for it
    // per level and slot: [level * cap + slot]
    float4* node_L;        // partial sum of the node
    float4* node_mul;      // f.rgb, |cos| / pdf of the ray that led to this node
    float4* node_hit;      // hit record of the node's surface
    float4* node_rd;       // incoming ray direction, bits(stage)
    uint32_t* node_inst;   // instanced scenes: the instance of the node's hit (0xffffffff = none)
    // textured scenes: the differential of the ray in flight (3 float4 per slot: rx_origin, ry_origin, rx_direction, ry_direction; the
    // flag says whether it has one) and of the ray that led to each node (for the node's transmission ray later on)
    float4* cur_diff;
    uint32_t* cur_has_diff;
    float4* node_diff;
    uint32_t* node_has_diff;
    // per slot and light sample: [slot * n_nee + q]
    float4* nee_a;         // light-strategy term pending the shadow ray, MIS weight of the BSDF strategy
    float4* nee_mf;        // f * |cos| of the BSDF strategy, scattering pdf
    float4* nee_md;        // its direction, bits(light)
    uint32_t* nee_flags;   // 1: shadow ray in flight, 2: MIS ray in flight, 4: fallback sample (no division by n_samples)
    uint32_t* nee_occl;    // written by k_trace
    float4* nee_mis_hit;   // written by k_trace
};

struct DSamplerCtx {
    const DRender* rp;
    SobolCtx sob;          // sob.index: the camera sample's index
    uint32_t array_end;
};
PB_D float ds_dimension(DSamplerCtx& S, uint32_t dim) {
    if (S.rp->halton) {  // HaltonSampler::sample_dimension panics past PRIME_TABLE_SIZE dimensions (halton.rs:256-262): flagged like Sobol's 1024, the render is refused
        if (dim >= (uint32_t)PB_HALTON_DIMS) { S.sob.overflow = true; return 0.0f; }
        return halton_sample_dimension(*S.rp, S.sob.index, dim);
    }
    if (dim >= 1024u) { S.sob.overflow = true; return 0.0f; }
    return sobol_sample_nib(S.sob, dim);
}
// GlobalSampler::get_1d / get_2d (sampler.rs): the dimensions of the 2D arrays are skipped
PB_D float ds_get_1d(DSamplerCtx& S, uint32_t& dim) {
    if (dim >= 5u && dim < S.array_end) dim = S.array_end;
    const float r = ds_dimension(S, dim);
    dim += 1u;
    return r;
}
PB_D float2 ds_get_2d(DSamplerCtx& S, uint32_t& dim) {
    if (dim + 1u >= 5u && dim < S.array_end) dim = S.array_end;
    const float y = ds_dimension(S, dim + 1u);
    const float x = ds_dimension(S, dim);
    dim += 2u;
    return make_float2(x, y);
}

PB_D BsdfFrame direct_frame(const DScene& sc, const DPaths& ps, uint32_t slot, const Isect& is) {
    BsdfFrame B;
    B.mat = sc.materials + is.material;
    if (B.mat->cls & PB_MAT_TEXTURED) B.mat = ps.slot_mat + slot;  // the lobes of this hit (direct_material below)
    B.ns = is.ns;
    B.ng = is.n;
    B.ss = norm3(is.sh_dpdu);
    B.ts = cross3(is.ns, B.ss);
    return B;
}
struct RayDiff { bool has; V3 rxo, ryo, rxd, ryd; };
PB_D RayDiff load_diff(const float4* __restrict__ q, bool has) {
    RayDiff d;
    d.has = has;
    const float4 q0 = q[0], q1 = q[1], q2 = q[2];
    d.rxo = mk3(q0.x, q0.y, q0.z); d.ryo = mk3(q0.w, q1.x, q1.y); d.rxd = mk3(q1.z, q1.w, q2.x); d.ryd = mk3(q2.y, q2.z, q2.w);
    return d;
}
PB_D void store_diff(float4* __restrict__ q, const RayDiff& d) {
    q[0] = make_float4(d.rxo.x, d.rxo.y, d.rxo.z, d.ryo.x);
    q[1] = make_float4(d.ryo.y, d.ryo.z, d.rxd.x, d.rxd.y);
    q[2] = make_float4(d.rxd.z, d.ryd.x, d.ryd.y, d.ryd.z);
}
// compute_scattering_functions of a node in a textured scene: compute_differentials against the incoming ray's differential, then,
// for a material with textures, its bump map / textures / lobe list of this hit into DPaths.slot_mat[slot] (`is` leaves with the
// bump-mapped shading frame).
PB_D UvDiff direct_material(const DScene& sc, const DPaths& ps, uint32_t slot, Isect& is, const RayDiff& rd) {
    UvDiff dd;
    dd.dudx = dd.dvdx = dd.dudy = dd.dvdy = 0.0f;
    dd.dpdx = dd.dpdy = mk3(0.0f, 0.0f, 0.0f);
    if (!sc.n_textures) return dd;
    if (rd.has) dd = compute_differentials(is, rd.rxo, rd.ryo, rd.rxd, rd.ryd);
    if (sc.materials[is.material].cls & PB_MAT_TEXTURED) {
        DMaterial m;
        bool bumped;
        material_at_hit(sc, is, dd, m, bumped, false);  // allow_multiple_lobes = false (directlighting.rs:77)
        ps.slot_mat[slot] = m;
    }
    return dd;
}

// The interaction of a hit and isect.wo, which both integrators use for everything (directlighting.rs:81, whitted.rs:58): -ray.d, or
// for a transformed instance hit the normalised vector carried back to world space (pb_interaction.cuh::hit_interaction).
PB_D Isect direct_isect(const DScene& sc, const DRender& rp, float4 hit, uint32_t inst, V3 rd, V3& wo) {
    if (sc.n_instances) return hit_interaction(sc, rp.instancing, (uint32_t)__float_as_int(hit.x), hit.y, hit.z, hit.w, inst, rd, wo);
    wo = -rd;
    return tri_interaction(sc, (uint32_t)__float_as_int(hit.x), hit.y, hit.z, hit.w);
}

// specular_reflect / specular_transmit up to the recursive call (directlighting.rs:124-260): true = a child ray was spawned.  In a
// textured scene the child's ray differential (:148-172, :219-249) goes into cur_diff.
PB_D bool direct_specular(const DScene& sc, const DPaths& ps, const DDirect& dd, DSamplerCtx& S, uint32_t& dim, uint32_t slot, int depth, const Isect& is, V3 wo,
                          bool transmit, const RayDiff& rdiff, const UvDiff& uvd, float4& r0, float4& r1) {
    const BsdfFrame B = direct_frame(sc, ps, slot, is);
    V3 wi = mk3(0.0f, 0.0f, 0.0f);
    float pdf = 0.0f;
    int st = 0;
    const float2 u = ds_get_2d(S, dim);
    const int flags = (transmit ? BSDF_TRANSMISSION : BSDF_REFLECTION) | BSDF_SPECULAR;
    const Sp f = bsdf_sample_f(B, wo, wi, u, pdf, flags, st);
    if (pdf > 0.0f && !is_black(f) && absdot3(wi, is.ns) != 0.0f) {
        const V3 o = offset_ray_origin(is.p, is.p_error, is.n, wi);
        r0 = make_float4(o.x, o.y, o.z, __int_as_float(0x7f800000));
        r1 = make_float4(wi.x, wi.y, wi.z, __uint_as_float(slot | (RAY_EXTEND << 30)));
        dd.node_mul[(size_t)(depth + 1) * dd.cap + slot] = make_float4(f.r, f.g, f.b, absdot3(wi, is.ns) / pdf);
        if (sc.n_textures) {
            dd.cur_has_diff[slot] = rdiff.has ? 1u : 0u;
            if (rdiff.has) {
                const V3 ns = is.ns;
                const V3 dndx = is.sh_dndu * uvd.dudx + is.sh_dndv * uvd.dvdx, dndy = is.sh_dndu * uvd.dudy + is.sh_dndv * uvd.dvdy;
                const V3 dwodx = -rdiff.rxd - wo, dwody = -rdiff.ryd - wo;
                const float ddndx = dot3(dwodx, ns) + dot3(wo, dndx), ddndy = dot3(dwody, ns) + dot3(wo, dndy);
                RayDiff c;
                c.has = true;
                c.rxo = is.p + uvd.dpdx;
                c.ryo = is.p + uvd.dpdy;
                if (!transmit) {
                    c.rxd = wi - dwodx + (dndx * dot3(wo, ns) + ns * ddndx) * 2.0f;
                    c.ryd = wi - dwody + (dndy * dot3(wo, ns) + ns * ddndy) * 2.0f;
                } else {
                    float eta = B.mat->eta;
                    const V3 w = -wo;
                    if (dot3(wo, ns) < 0.0f) eta = 1.0f / eta;
                    const float mu = eta * dot3(w, ns) - dot3(wi, ns);
                    const float dmudx = (eta - (eta * eta * dot3(w, ns)) / dot3(wi, ns)) * ddndx;
                    const float dmudy = (eta - (eta * eta * dot3(w, ns)) / dot3(wi, ns)) * ddndy;
                    c.rxd = wi + dwodx * eta - (dndx * mu + ns * dmudx);
                    c.ryd = wi + dwody * eta - (dndy * mu + ns * dmudy);
                }
                store_diff(dd.cur_diff + 3 * (size_t)slot, c);
            }
        }
        return true;
    }
    return false;
}

// The first iteration's start of every camera sample, for camera rays WITHOUT a differential (the environment camera,
// environment.rs:106: its first hits look textures up at level 0, like any later ray's): what k_direct_step does when `first` is set,
// but with cur_has_diff = 0.  k_direct_step then runs its first iteration with first = 0 and reads this state.  (A second
// instantiation of k_direct_step would have done the same, but it changes the compiler's inlining of the texture code shared with
// k_texture and the alpha-tested k_trace, and with it their code.)
__global__ void __launch_bounds__(128) k_direct_start_nodiff(DScene sc, DPaths ps, DDirect dd, BatchInfo bi) {
    const uint32_t slot = blockIdx.x * blockDim.x + threadIdx.x;
    if (slot >= bi.n_pixels * bi.n_samples) return;
    const uint32_t state = (__float_as_uint(ps.L[slot].w) & PF_HAS_RAY) ? DS_WAIT_TRACE : DS_DONE;
    dd.state[slot] = state;
    dd.depth[slot] = 0;
    dd.arr_off[slot] = 0u;
    dd.nee_depth[slot] = -1;
    if (sc.n_textures) dd.cur_has_diff[slot] = 0u;
    if (state == DS_DONE) ps.L[slot] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
}

__global__ void __launch_bounds__(128) k_direct_step(DScene sc, DRender rp, DPaths ps, DDirect dd, BatchInfo bi, const uint32_t* __restrict__ nib, uint32_t first,
                                                     float4* __restrict__ rays, uint32_t* __restrict__ d_nrays, uint32_t* __restrict__ d_active,
                                                     uint32_t* __restrict__ d_error, const uint32_t* __restrict__ prev_active) {
    // an iteration the host queued before it knew that the previous one had left nothing to do (pbrt_gpu.cu, late-polled loop)
    if (prev_active && *prev_active == 0u) return;
    const uint32_t n_paths = bi.n_pixels * bi.n_samples;
    const uint32_t slot = blockIdx.x * blockDim.x + threadIdx.x;
    float4 r0 = make_float4(0.0f, 0.0f, 0.0f, 0.0f), r1 = r0;
    bool emit = false, live = false;
    if (slot < n_paths) {
        uint32_t state = dd.state[slot];
        if (first) {
            state = (__float_as_uint(ps.L[slot].w) & PF_HAS_RAY) ? DS_WAIT_TRACE : DS_DONE;
            dd.depth[slot] = 0;
            dd.arr_off[slot] = 0u;
            dd.nee_depth[slot] = -1;
            if (sc.n_textures) {  // the camera ray's differential (k_raygen)
                dd.cur_has_diff[slot] = 1u;
                for (int k = 0; k < 3; ++k) dd.cur_diff[3 * (size_t)slot + k] = ps.ray_diff[3 * (size_t)slot + k];
            }
            if (state == DS_DONE) ps.L[slot] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        }
        dd.fresh[slot] = 0u;
        if (state != DS_DONE) {
            const uint2 si = ps.sobol[slot];
            DSamplerCtx S;
            S.rp = &rp;
            S.sob.nib = nib; S.sob.stride = PB_SOBOL_CHUNKS; S.sob.n_chunks = dd.n_chunks; S.sob.dim = 0; S.sob.overflow = false;
            S.sob.index = ((uint64_t)si.y << 32) | si.x;
            S.array_end = dd.array_end;
            uint32_t dim = ps.dim[slot];
            int depth = dd.depth[slot];
            // ---- (1) fold the direct light of the node shaded in the previous iteration ----
            const int nd = dd.nee_depth[slot];
            if (nd >= 0) {
                const float4 nl = dd.node_L[(size_t)nd * dd.cap + slot];
                Sp l = mksp(nl.x, nl.y, nl.z);
                Sp all = sp1(0.0f);       // uniform_sample_all_lights' own accumulator
                Sp ld_light = sp1(0.0f);  // the per-light sum over its samples
                for (uint32_t q = 0; q < dd.n_nee; ++q) {
                    const size_t r = (size_t)slot * dd.n_nee + q;
                    const uint32_t fl = dd.nee_flags[r];
                    const uint32_t j = dd.nee_light[q], k = dd.nee_k[q];
                    Sp ld = sp1(0.0f);    // estimate_direct's return value
                    const float4 a = dd.nee_a[r];
                    if ((fl & 1u) && dd.nee_occl[r] == 0u) ld = ld + mksp(a.x, a.y, a.z);
                    if (fl & 2u) {
                        const float4 mh = dd.nee_mis_hit[r], md = dd.nee_md[r], mf = dd.nee_mf[r];
                        const int mprim = __float_as_int(mh.x);
                        const uint32_t light_num = __float_as_uint(md.w);
                        if (mprim >= 0) {
                            V3 lp, ln;
                            int hit_light;
                            tri_point_normal(sc, (uint32_t)mprim, mh.y, mh.z, mh.w, lp, ln, hit_light);
                            if (hit_light == (int)light_num) {
                                const Sp le = light_L(sc.lights[light_num], ln, -mk3(md.x, md.y, md.z));
                                if (!is_black(le)) ld = ld + mksp(mf.x, mf.y, mf.z) * le * sp1(1.0f) * a.w / mf.w;
                            }
                        } else if (sc.n_inf) {
                            const Sp le = light_le(sc, sc.lights[light_num], mk3(md.x, md.y, md.z));
                            if (!is_black(le)) ld = ld + mksp(mf.x, mf.y, mf.z) * le * sp1(1.0f) * a.w / mf.w;
                        }
                    }
                    if (dd.whitted) {
                        l = l + ld;  // whitted.rs:93: straight into l, light by light (ld is the one unoccluded term or black)
                    } else if (!dd.sample_all) {
                        if (fl & 8u) l = l + ld / (1.0f / (float)sc.n_lights);  // estimate_direct(..) / pdf, integrator.rs:388,402
                    } else {
                        if (fl & 4u) {  // fallback: one sample, no division (integrator.rs:316-329); only k == 0 carries it
                            if (k == 0u) all = all + ld;
                        } else {
                            if (k == 0u) ld_light = sp1(0.0f);
                            ld_light = ld_light + ld;
                            if (k + 1u == dd.light_n[j]) all = all + ld_light / (float)dd.light_n[j];
                        }
                    }
                }
                if (!dd.whitted && dd.sample_all) l = l + all;
                dd.node_L[(size_t)nd * dd.cap + slot] = make_float4(l.r, l.g, l.b, 0.0f);
                dd.nee_depth[slot] = -1;
            }
            // ---- (2) the ray that was traced, or a node that only waited for its direct light ----
            bool returning = false;
            if (state == DS_WAIT_TRACE) {
                const float4 hit = ps.hit[slot];
                const int prim = __float_as_int(hit.x);
                const float4 rd4 = ps.ray_d[slot];
                const V3 rd = mk3(rd4.x, rd4.y, rd4.z);
                if (prim < 0) {  // light.le(ray) of every light: zero unless infinite
                    Sp l = sp1(0.0f);
                    for (uint32_t k = 0; k < sc.n_lights; ++k) l = l + light_le(sc, sc.lights[k], rd);
                    dd.node_L[(size_t)depth * dd.cap + slot] = make_float4(l.r, l.g, l.b, 0.0f);
                    returning = true;
                } else {
                    const uint32_t inst = sc.n_instances ? ps.hit_inst[slot] : 0xffffffffu;
                    V3 wo;
                    Isect is = direct_isect(sc, rp, hit, inst, rd, wo);
                    if (is.material == 0xffffffffu) {  // no BSDF: continue through the surface at the same depth
                        const V3 o = offset_ray_origin(is.p, is.p_error, is.n, rd);
                        r0 = make_float4(o.x, o.y, o.z, __int_as_float(0x7f800000));
                        r1 = make_float4(rd.x, rd.y, rd.z, __uint_as_float(slot | (RAY_EXTEND << 30)));
                        emit = true;
                        if (sc.n_textures) dd.cur_has_diff[slot] = 0u;  // isect.spawn_ray(ray.d) carries no differential
                    } else {
                        RayDiff rdiff;
                        rdiff.has = false;
                        if (sc.n_textures) {  // the incoming ray's differential: kept with the node for its transmission ray later on
                            rdiff = load_diff(dd.cur_diff + 3 * (size_t)slot, dd.cur_has_diff[slot] != 0u);
                            dd.node_has_diff[(size_t)depth * dd.cap + slot] = rdiff.has ? 1u : 0u;
                            if (rdiff.has) store_diff(dd.node_diff + 3 * ((size_t)depth * dd.cap + slot), rdiff);
                        }
                        const UvDiff uvd = direct_material(sc, ps, slot, is, rdiff);
                        if (sc.n_textures) {  // k_direct_nee shades with the (possibly bump-mapped) frame of this hit
                            ps.slot_frame[2 * (size_t)slot] = make_float4(is.ns.x, is.ns.y, is.ns.z, 0.0f);
                            ps.slot_frame[2 * (size_t)slot + 1] = make_float4(is.sh_dpdu.x, is.sh_dpdu.y, is.sh_dpdu.z, 0.0f);
                        }
                        Sp l = sp1(0.0f);
                        if (is.area_light >= 0) l = l + light_L(sc.lights[is.area_light], is.n, wo);
                        dd.node_L[(size_t)depth * dd.cap + slot] = make_float4(l.r, l.g, l.b, 0.0f);
                        dd.node_hit[(size_t)depth * dd.cap + slot] = hit;
                        if (sc.n_instances) dd.node_inst[(size_t)depth * dd.cap + slot] = inst;
                        // direct light: the draws happen in k_direct_nee; here only the sampler state moves past them
                        if (sc.n_lights) {
                            dd.nee_depth[slot] = depth;
                            dd.nee_dim[slot] = dim;
                            const uint32_t a0 = dd.arr_off[slot];
                            dd.nee_arr[slot] = a0;
                            dd.fresh[slot] = 1u;
                            if (dd.whitted) {
                                for (uint32_t k = 0; k < sc.n_lights; ++k) (void)ds_get_2d(S, dim);
                            } else if (!dd.sample_all) {
                                (void)ds_get_1d(S, dim); (void)ds_get_2d(S, dim); (void)ds_get_2d(S, dim);
                            } else {
                                const uint32_t j0 = min(sc.n_lights, (dd.n_arrays - min(a0, dd.n_arrays)) / 2u);  // lights served from the arrays
                                dd.arr_off[slot] = a0 + 2u * j0;
                                for (uint32_t k = j0; k < sc.n_lights; ++k) { (void)ds_get_2d(S, dim); (void)ds_get_2d(S, dim); }
                            }
                        }
                        uint32_t stage = STAGE_NONE;
                        state = DS_COMPLETE_PENDING;
                        if ((uint32_t)(depth + 1) < dd.max_depth) {
                            if (direct_specular(sc, ps, dd, S, dim, slot, depth, is, wo, false, rdiff, uvd, r0, r1)) {
                                stage = STAGE_AFTER_REFLECT; emit = true;
                            } else if (direct_specular(sc, ps, dd, S, dim, slot, depth, is, wo, true, rdiff, uvd, r0, r1)) {
                                stage = STAGE_AFTER_TRANSMIT; emit = true;
                            }
                        }
                        dd.node_rd[(size_t)depth * dd.cap + slot] = make_float4(rd.x, rd.y, rd.z, __uint_as_float(stage));
                        if (emit) { depth += 1; state = DS_WAIT_TRACE; }
                        else if (!sc.n_lights) returning = true;  // nothing in flight for this node: it is complete now
                    }
                }
            } else returning = true;  // DS_COMPLETE_PENDING: its direct light has just been folded
            // ---- (3) return through finished nodes ----
            while (returning) {
                const float4 ld4 = dd.node_L[(size_t)depth * dd.cap + slot];
                if (depth == 0) {
                    ps.L[slot] = make_float4(ld4.x, ld4.y, ld4.z, 0.0f);
                    state = DS_DONE;
                    break;
                }
                const float4 mul = dd.node_mul[(size_t)depth * dd.cap + slot];
                const int p = depth - 1;
                const float4 pl4 = dd.node_L[(size_t)p * dd.cap + slot];
                // l += f * li(child) * Spectrum(|cos| / pdf)
                const Sp pl = mksp(pl4.x, pl4.y, pl4.z) + mksp(mul.x, mul.y, mul.z) * mksp(ld4.x, ld4.y, ld4.z) * sp1(mul.w);
                dd.node_L[(size_t)p * dd.cap + slot] = make_float4(pl.r, pl.g, pl.b, 0.0f);
                depth = p;
                const float4 prd = dd.node_rd[(size_t)p * dd.cap + slot];
                if (__float_as_uint(prd.w) == STAGE_AFTER_REFLECT) {  // the parent's specular_transmit comes next
                    const float4 ph = dd.node_hit[(size_t)p * dd.cap + slot];
                    const V3 rd = mk3(prd.x, prd.y, prd.z);
                    V3 pwo;
                    Isect is = direct_isect(sc, rp, ph, sc.n_instances ? dd.node_inst[(size_t)p * dd.cap + slot] : 0xffffffffu, rd, pwo);
                    RayDiff pdiff;
                    pdiff.has = false;
                    if (sc.n_textures) pdiff = load_diff(dd.node_diff + 3 * ((size_t)p * dd.cap + slot), dd.node_has_diff[(size_t)p * dd.cap + slot] != 0u);
                    const UvDiff puvd = direct_material(sc, ps, slot, is, pdiff);  // the node's material again: deeper nodes have used slot_mat since
                    if (direct_specular(sc, ps, dd, S, dim, slot, p, is, pwo, true, pdiff, puvd, r0, r1)) {
                        dd.node_rd[(size_t)p * dd.cap + slot] = make_float4(prd.x, prd.y, prd.z, __uint_as_float(STAGE_AFTER_TRANSMIT));
                        depth = p + 1;
                        emit = true;
                        state = DS_WAIT_TRACE;
                        break;
                    }
                }
            }
            if (emit) ps.ray_d[slot] = make_float4(r1.x, r1.y, r1.z, 0.0f);
            ps.dim[slot] = dim;
            dd.depth[slot] = depth;
            if (S.sob.overflow) atomicOr(d_error, 1u);
        }
        dd.state[slot] = state;
        live = state != DS_DONE;
    }
    const uint32_t pos = queue_append(d_nrays, emit);
    if (emit) { rays[2 * (size_t)pos] = r0; rays[2 * (size_t)pos + 1] = r1; }
    const uint32_t n_live = warp_sum(live ? 1u : 0u);  // camera samples that still need an iteration (the host's loop condition)
    if ((threadIdx.x & 31) == 0 && n_live) atomicAdd(d_active, n_live);
}

// estimate_direct (integrator.rs:406-570) for light sample q of the node shaded in this iteration, up to its two rays
template <int LIGHTS>
__global__ void __launch_bounds__(128) k_direct_nee(DScene sc, DRender rp, DPaths ps, DDirect dd, BatchInfo bi, const uint32_t* __restrict__ nib,
                                                    const uint64_t* __restrict__ vdc, const uint64_t* __restrict__ vdci, float4* __restrict__ rays,
                                                    uint32_t* __restrict__ d_nrays, DCounters* cnt, uint32_t* __restrict__ d_error,
                                                    const uint32_t* __restrict__ prev_active) {
    if (prev_active && *prev_active == 0u) return;  // see k_direct_step: the `fresh` flags are stale then
    __shared__ uint64_t s_vdc[52], s_vdci[52];
    if (threadIdx.x < 52) {
        const uint32_t m = rp.log2_res;
        s_vdc[threadIdx.x] = m ? vdc[(m - 1) * 52 + threadIdx.x] : 0;
        s_vdci[threadIdx.x] = m ? vdci[(m - 1) * 52 + threadIdx.x] : 0;
    }
    __syncthreads();
    const uint32_t n_paths = bi.n_pixels * bi.n_samples;
    const uint64_t total = (uint64_t)n_paths * dd.n_nee;
    const uint64_t gid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    float4 sh0 = make_float4(0.0f, 0.0f, 0.0f, 0.0f), sh1 = sh0, mis0 = sh0, mis1 = sh0;
    bool emit_sh = false, emit_mis = false;
    uint32_t n_light_tests = 0;
    if (gid < total) {
        const uint32_t slot = (uint32_t)(gid / dd.n_nee), q = (uint32_t)(gid % dd.n_nee);
        if (dd.fresh[slot]) {
            const int depth = dd.nee_depth[slot];
            const float4 hit = dd.node_hit[(size_t)depth * dd.cap + slot];
            const float4 rd4 = dd.node_rd[(size_t)depth * dd.cap + slot];
            V3 wo;
            Isect is = direct_isect(sc, rp, hit, sc.n_instances ? dd.node_inst[(size_t)depth * dd.cap + slot] : 0xffffffffu, mk3(rd4.x, rd4.y, rd4.z), wo);
            const V3 ns_before_bump = is.ns;  // whitted.rs:58 reads shading.n before compute_scattering_functions runs the bump map
            if (sc.n_textures) {  // the frame k_direct_step left for this hit (bump maps)
                const float4 f0 = ps.slot_frame[2 * (size_t)slot], f1 = ps.slot_frame[2 * (size_t)slot + 1];
                is.ns = mk3(f0.x, f0.y, f0.z);
                is.sh_dpdu = mk3(f1.x, f1.y, f1.z);
            }
            const BsdfFrame B = direct_frame(sc, ps, slot, is);
            const uint2 si = ps.sobol[slot];
            DSamplerCtx S;
            S.rp = &rp;
            S.sob.nib = nib; S.sob.stride = PB_SOBOL_CHUNKS; S.sob.n_chunks = dd.n_chunks; S.sob.dim = 0; S.sob.overflow = false;
            S.sob.index = ((uint64_t)si.y << 32) | si.x;
            S.array_end = dd.array_end;
            uint32_t dim = dd.nee_dim[slot];
            uint32_t light_num = dd.nee_light[q];
            const uint32_t k = dd.nee_k[q];
            float2 u_light = make_float2(0.0f, 0.0f), u_scat = u_light;
            uint32_t flags = 0u;
            bool active = true;
            if (dd.whitted) {
                for (uint32_t j = 0; j < light_num; ++j) (void)ds_get_2d(S, dim);
                u_light = ds_get_2d(S, dim);
            } else if (!dd.sample_all) {
                const float u1 = ds_get_1d(S, dim);
                light_num = min((uint32_t)f2i_sat(u1 * (float)sc.n_lights), sc.n_lights - 1u);
                u_light = ds_get_2d(S, dim);
                u_scat = ds_get_2d(S, dim);
                flags |= 8u;
            } else {
                const uint32_t a0 = dd.nee_arr[slot];
                const uint32_t j0 = min(sc.n_lights, (dd.n_arrays - min(a0, dd.n_arrays)) / 2u);
                if (light_num < j0) {  // entry s_pix * n + k of the arrays a0 + 2j (u_light) and a0 + 2j + 1 (u_scattering)
                    const uint32_t n = dd.light_n[light_num];
                    const uint32_t pl = slot / bi.n_samples, s_pix = bi.first_sample + slot % bi.n_samples;
                    const uint32_t pix = bi.first_pixel + pl;
                    int px, py;
                    share_pixel(rp, pix, px, py);
                    const uint64_t jn = (uint64_t)s_pix * n + k;
                    DSamplerCtx A = S;
                    A.sob.index = rp.halton ? halton_index(rp, px, py, jn) : sobol_interval_to_index(s_vdc, s_vdci, rp.log2_res, jn, px - rp.sb[0], py - rp.sb[1]);
                    const uint32_t dl = 5u + 2u * (a0 + 2u * light_num), dsx = dl + 2u;
                    u_light = make_float2(ds_dimension(A, dl), ds_dimension(A, dl + 1u));
                    u_scat = make_float2(ds_dimension(A, dsx), ds_dimension(A, dsx + 1u));
                    if (A.sob.overflow) S.sob.overflow = true;
                } else {  // the arrays are used up: one regular sample for this light
                    flags |= 4u;
                    if (k != 0u) active = false;
                    else {
                        for (uint32_t j = j0; j < light_num; ++j) { (void)ds_get_2d(S, dim); (void)ds_get_2d(S, dim); }
                        u_light = ds_get_2d(S, dim);
                        u_scat = ds_get_2d(S, dim);
                    }
                }
            }
            const size_t r = (size_t)slot * dd.n_nee + q;
            Sp a = sp1(0.0f);
            float mis_w = 0.0f;
            if (active) {
                const DLight& light = sc.lights[light_num];
                V3 wi = mk3(0.0f, 0.0f, 0.0f);
                float light_pdf = 0.0f, scattering_pdf = 0.0f;
                LightSample ls;
                const Sp li = light_sample_li<LIGHTS>(sc, light, is.p, u_light, wi, light_pdf, ls);
                if (dd.whitted) {  // whitted.rs:84-96
                    if (!(is_black(li) || light_pdf == 0.0f)) {
                        const Sp f = bsdf_f(B, wo, wi, BSDF_ALL);
                        if (!is_black(f)) {
                            const V3 origin = offset_ray_origin(is.p, is.p_error, is.n, ls.p - is.p);
                            const V3 target = offset_ray_origin(ls.p, ls.p_error, ls.n, origin - ls.p);
                            const V3 sd = target - origin;
                            a = f * li * absdot3(wi, ns_before_bump) / light_pdf;
                            sh0 = make_float4(origin.x, origin.y, origin.z, 1.0f - PB_SHADOW_EPSILON);
                            sh1 = make_float4(sd.x, sd.y, sd.z, __uint_as_float((uint32_t)r | (RAY_SHADOW << 30)));
                            emit_sh = true;
                            flags |= 1u;
                        }
                    }
                } else {
                    const int NONSPEC = BSDF_ALL & ~BSDF_SPECULAR;
                    if (light_pdf > 0.0f && !is_black(li)) {
                        const Sp f = bsdf_f(B, wo, wi, NONSPEC) * sp1(absdot3(wi, is.ns));
                        scattering_pdf = bsdf_pdf(B, wo, wi, NONSPEC);
                        if (!is_black(f)) {
                            const V3 origin = offset_ray_origin(is.p, is.p_error, is.n, ls.p - is.p);
                            const V3 target = offset_ray_origin(ls.p, ls.p_error, ls.n, origin - ls.p);
                            const V3 sd = target - origin;
                            if (light_is_delta<LIGHTS>(light)) a = f * li / light_pdf;
                            else a = f * li * sp1(power_heuristic(light_pdf, scattering_pdf)) / light_pdf;
                            sh0 = make_float4(origin.x, origin.y, origin.z, 1.0f - PB_SHADOW_EPSILON);
                            sh1 = make_float4(sd.x, sd.y, sd.z, __uint_as_float((uint32_t)r | (RAY_SHADOW << 30)));
                            emit_sh = true;
                            flags |= 1u;
                        }
                    }
                    if (!light_is_delta<LIGHTS>(light)) {
                        int st = 0;
                        Sp f2 = bsdf_sample_f(B, wo, wi, u_scat, scattering_pdf, NONSPEC, st);
                        f2 = f2 * sp1(absdot3(wi, is.ns));
                        if (!is_black(f2) && scattering_pdf > 0.0f) {
                            const V3 mo = offset_ray_origin(is.p, is.p_error, is.n, wi);
                            if (light.kind == 0u) n_light_tests++;
                            const float lp = light_pdf_li<LIGHTS>(sc, light, is.p, mo, wi);
                            if (lp != 0.0f) {
                                mis_w = power_heuristic(scattering_pdf, lp);
                                mis0 = make_float4(mo.x, mo.y, mo.z, __int_as_float(0x7f800000));
                                mis1 = make_float4(wi.x, wi.y, wi.z, __uint_as_float((uint32_t)r | (RAY_MIS << 30)));
                                emit_mis = true;
                                dd.nee_md[r] = make_float4(wi.x, wi.y, wi.z, __uint_as_float(light_num));
                                dd.nee_mf[r] = make_float4(f2.r, f2.g, f2.b, scattering_pdf);
                                flags |= 2u;
                            }
                        }
                    }
                }
            }
            dd.nee_a[r] = make_float4(a.r, a.g, a.b, mis_w);
            dd.nee_flags[r] = flags;
            if (S.sob.overflow) atomicOr(d_error, 1u);
        }
    }
    const uint32_t p0 = queue_append(d_nrays, emit_sh);
    if (emit_sh) { rays[2 * (size_t)p0] = sh0; rays[2 * (size_t)p0 + 1] = sh1; }
    const uint32_t p1 = queue_append(d_nrays, emit_mis);
    if (emit_mis) { rays[2 * (size_t)p1] = mis0; rays[2 * (size_t)p1 + 1] = mis1; }
    const uint32_t tot = warp_sum(n_light_tests);
    if ((threadIdx.x & 31) == 0 && tot) atomicAdd(&cnt->light_tri_tests, (unsigned long long)tot);
}

}  // namespace pb
