// pbrt_gpu.cu -- C ABI (include/pbrt_gpu.h) over the wavefront kernels.
// Host side: flatten the caller's scene into the HBM layout of pb_scene.cuh, drive the per-batch
// kernel sequence, and hand back FilmTilePixel-compatible {contrib_sum, filter_weight_sum}.
// There is deliberately NO CPU fallback: without a usable device every entry point fails.
#include <sched.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <atomic>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../include/pbrt_gpu.h"
#include "pb_kernels.cuh"
#include "pb_direct.cuh"

using namespace pb;

extern "C" {
extern const unsigned char pb_sobol_blob_start[];
extern const unsigned char pb_sobol_blob_end[];
}

namespace {

thread_local std::string g_err;
std::atomic<unsigned long long> g_launches{0};

int fail(int code, const std::string& msg) { g_err = msg; return code; }
#define CK(call)                                                                                         \
    do {                                                                                                 \
        cudaError_t e_ = (call);                                                                         \
        if (e_ != cudaSuccess) return fail(PBRT_E_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_)); \
    } while (0)

// Device allocations that come and go with a scene are recycled through a per-device free list instead of going back to the driver:
// a caller that re-creates the scene for every frame then makes no cudaMalloc / cudaFree call at all in the steady state.  Those calls
// take the driver's allocation lock, and anything else on the box that holds it -- a monitoring tool polling the GPU once a second
// was enough -- stalled some scene_create calls for a large fraction of a second.
struct BufCache {
    std::mutex mu;
    std::multimap<size_t, void*> free_list;  // capacity in bytes -> block
    size_t bytes = 0;
    static constexpr size_t cap = (size_t)6 << 30;
    void* get(size_t want, size_t& got) {
        std::lock_guard<std::mutex> g(mu);
        // exact sizes only: the buffers of a re-created scene repeat to the byte, and a "close enough" block handed to the wrong
        // request left the right one to cudaMalloc -- the very call this cache exists to avoid
        auto it = free_list.find(want);
        if (it == free_list.end()) return nullptr;
        void* p = it->second;
        got = it->first;
        bytes -= it->first;
        free_list.erase(it);
        return p;
    }
    bool put(void* p, size_t n) {
        std::lock_guard<std::mutex> g(mu);
        if (bytes + n > cap) return false;
        free_list.emplace(n, p);
        bytes += n;
        return true;
    }
};
static BufCache* buf_cache(int device) {
    static BufCache* pool[64] = {nullptr};
    static std::mutex mu;
    std::lock_guard<std::mutex> g(mu);
    if (device < 0 || device >= 64) return nullptr;
    if (!pool[device]) pool[device] = new BufCache();  // lives until process exit
    return pool[device];
}

template <typename T> struct DevBuf {
    T* p = nullptr;
    size_t n = 0;
    int cache_dev = -1;  // >= 0: recycle through that device's BufCache (scene buffers)
    ~DevBuf() { release(); }
    void release() {
        if (p) {
            BufCache* c = cache_dev >= 0 ? buf_cache(cache_dev) : nullptr;
            if (!c || !c->put(p, n * sizeof(T))) cudaFree(p);
        }
        p = nullptr; n = 0;
    }
    cudaError_t alloc(size_t count) {
        if (p && n >= count) return cudaSuccess;
        release();
        if (count == 0) return cudaSuccess;
        if (BufCache* c = cache_dev >= 0 ? buf_cache(cache_dev) : nullptr) {
            size_t got = 0;
            if (void* q = c->get(count * sizeof(T), got)) { p = static_cast<T*>(q); n = got / sizeof(T); return cudaSuccess; }
        }
        cudaError_t e = cudaMalloc((void**)&p, count * sizeof(T));
        if (e == cudaSuccess) n = count;
        return e;
    }
    cudaError_t upload(const std::vector<T>& h) {
        cudaError_t e = alloc(h.size());
        if (e != cudaSuccess || h.empty()) return e;
        return cudaMemcpy(p, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice);
    }
};

// ---- material -> lobe list: pb_material.cuh (shared with k_texture, which compiles textured materials per hit) ----
float roughness_to_alpha(float roughness) {  // microfacet.rs:243-255
    if (1e-3f > roughness) roughness = 1e-3f;
    float x = logf(roughness);
    return 1.62142f + 0.819955f * x + 0.1734f * x * x + 0.0171201f * x * x * x + 0.000640711f * x * x * x * x;
}
// The two Trowbridge-Reitz alphas of a material: its roughness parameters through roughness_to_alpha when "remaproughness" is set.
// They never depend on a texture here (float parameters are constants), so the device-side compile takes them from the host.
void material_alphas(const PbrtMaterial& m, float& au, float& av) {
    const float* p = m.params;
    int iu = -1, iv = -1, ir = -1;
    switch (m.kind) {
        case PBRT_MAT_PLASTIC: iu = iv = 6; ir = 7; break;
        case PBRT_MAT_METAL: case PBRT_MAT_SUBSTRATE: iu = 6; iv = 7; ir = 8; break;
        case PBRT_MAT_GLASS: iu = 7; iv = 8; ir = 9; break;
        case PBRT_MAT_UBER: iu = 15; iv = 16; ir = 18; break;
        case PBRT_MAT_TRANSLUCENT: iu = iv = 12; ir = 13; break;
        default: break;
    }
    au = av = 0.0f;
    if (iu < 0) return;
    au = p[iu]; av = p[iv];
    if (p[ir] != 0.0f) { au = roughness_to_alpha(au); av = roughness_to_alpha(av); }
}
bool compile_material(const PbrtMaterial& m, DMaterial& out, bool allow_multiple_lobes = true) {
    float au, av;
    material_alphas(m, au, av);
    return compile_material_core(m.kind, m.params, au, av, out, allow_multiple_lobes);
}
// Material `index` of the caller's array, MixMaterial included (mixmat.rs:41-98; pbrt_gpu.h on PBRT_MAT_MIX): m1 compiled with scale
// s1 = clamp(amount), m2 with s2 = clamp(1 - s1), m2's lobes added to m1's.  `scale` is what a parent mix hands down: every other kind
// stores it in each lobe (sc_opt), a mix ignores it (`_scale`, mixmat.rs:48).  *why names what made the material unusable.
bool compile_material_at(const PbrtMaterial* mats, uint32_t n_mats, uint32_t index, DMaterial& out, bool allow_multiple_lobes, const Sp* scale, const char** why) {
    const PbrtMaterial& m = mats[index];
    if (m.kind != PBRT_MAT_MIX) {
        if (!compile_material(m, out, allow_multiple_lobes)) { *why = "material kind outside the GPU path"; return false; }
        if (scale) scale_lobes(out, *scale);
        return true;
    }
    const float i1 = m.params[3], i2 = m.params[4];
    if (!(i1 >= 0.0f && i1 < (float)index && i2 >= 0.0f && i2 < (float)index) || i1 != floorf(i1) || i2 != floorf(i2) || index >= n_mats) {
        *why = "MixMaterial: a child index is not a whole number below the mix's own index";
        return false;
    }
    if (m.bump) { *why = "MixMaterial has no bump map"; return false; }
    for (int g = 0; g < PBRT_MAX_TEX_GROUPS; ++g)
        if (m.tex[g]) { *why = "MixMaterial with a textured amount is outside the GPU path"; return false; }
    for (uint32_t c : {(uint32_t)i1, (uint32_t)i2}) {
        bool plain = mats[c].bump == 0;
        for (int g = 0; g < PBRT_MAX_TEX_GROUPS; ++g) plain = plain && mats[c].tex[g] == 0;
        if (!plain) { *why = "MixMaterial over a textured or bump-mapped material is outside the GPU path"; return false; }
    }
    const Sp s1 = clamp_pos(sp3(m.params));
    const Sp s2 = clamp_pos(sp1(1.0f) - s1);
    DMaterial second;
    if (!compile_material_at(mats, n_mats, (uint32_t)i1, out, allow_multiple_lobes, &s1, why)) return false;
    if (!compile_material_at(mats, n_mats, (uint32_t)i2, second, allow_multiple_lobes, &s2, why)) return false;
    if (!append_lobes(out, second)) { *why = "MixMaterial with more than five lobes in all is outside the GPU path"; return false; }
    return true;
}

// Distribution1D::new (sampling.rs:24-49) for the fixed (uniform / power) strategies
void make_distribution(const std::vector<float>& f, std::vector<float>& cdf, float& func_int) {
    size_t n = f.size();
    cdf.assign(n + 1, 0.0f);
    for (size_t i = 1; i <= n; ++i) cdf[i] = cdf[i - 1] + f[i - 1] / (float)n;
    func_int = cdf[n];
    if (func_int == 0.0f) for (size_t i = 1; i <= n; ++i) cdf[i] = (float)i / (float)n;
    else for (size_t i = 1; i <= n; ++i) cdf[i] /= func_int;
}
// InfiniteAreaLight construction on the host (lights/infinite.rs:250-300 and the image branches above it): the MIP pyramid
// of a power-of-two lat-long map (MipMap::new mipmap.rs:150-188, ImageWrap::Repeat), the scalar image lum * sin(theta) at twice
// the resolution and its Distribution2D (sampling.rs:150-183), and the texel that power() looks up (infinite.rs:349-355).
struct HostEnv {
    int w = 0, h = 0, nu = 0, nv = 0;
    std::vector<float4> texels;
    std::vector<float> cond_func, cond_cdf, cond_int, marg_func, marg_cdf;
    float marg_int = 0.0f;
    Sp power_L = sp1(0.0f);
};
struct MipLevel { int us, vs; std::vector<Sp> t; uint32_t wrap = PBRT_WRAP_REPEAT; };
static Sp mip_texel(const MipLevel& l, long s, long t) {  // mipmap.rs:208-232 (Black answers the clamped texel, like Clamp)
    if (l.wrap == PBRT_WRAP_REPEAT) return l.t[((size_t)t & (size_t)(l.vs - 1)) * l.us + ((size_t)s & (size_t)(l.us - 1))];
    const long ss = std::min(std::max(s, 0L), (long)l.us - 1), tt = std::min(std::max(t, 0L), (long)l.vs - 1);
    return l.t[(size_t)tt * l.us + (size_t)ss];
}
static Sp mip_triangle(const std::vector<MipLevel>& pyr, size_t level, float sx, float sy) {  // mipmap.rs:323-336
    if (level > pyr.size() - 1) level = pyr.size() - 1;
    const MipLevel& l = pyr[level];
    float s = sx * (float)l.us - 0.5f, t = sy * (float)l.vs - 0.5f;
    long s0 = (long)floorf(s), t0 = (long)floorf(t);
    float ds = s - (float)s0, dt = t - (float)t0;
    Sp a = mip_texel(l, s0 + 1, t0 + 1) * (ds * dt);
    Sp b = mip_texel(l, s0 + 1, t0) * (ds * (1.0f - dt));
    Sp c = mip_texel(l, s0, t0 + 1) * ((1.0f - ds) * dt);
    Sp d = mip_texel(l, s0, t0) * ((1.0f - ds) * (1.0f - dt));
    return d + c + b + a;
}
static Sp mip_lookup(const std::vector<MipLevel>& pyr, float sx, float sy, float width) {  // lookup_pnt_flt mipmap.rs:233-252
    const float n = (float)pyr.size();
    float level = n - 1.0f + log2f(fmaxf(width, 1e-8f));
    if (level < 0.0f) return mip_triangle(pyr, 0, sx, sy);
    if (level >= n - 1.0f) return mip_texel(pyr.back(), 0, 0);
    size_t il = (size_t)floorf(level);
    float delta = level - (float)il;
    return mip_triangle(pyr, il, sx, sy) * (1.0f - delta) + mip_triangle(pyr, il + 1, sx, sy) * delta;
}
static float lanczos_w(float x, float tau) {  // texture.rs:426-439
    x = fabsf(x);
    if (x < 1e-5f) return 1.0f;
    if (x > 1.0f) return 0.0f;
    x *= PB_PI;
    const float s = sinf(x * tau) / (x * tau);
    return s * (sinf(x) / x);
}
// MipMap::new's resampling of one axis to the next power of two (mipmap.rs:298-322): 4-tap Lanczos, normalised weights
struct AxisResample { std::vector<int> first; std::vector<float> w; };
static AxisResample resample_axis(int old_res, int new_res) {
    AxisResample a;
    a.first.resize(new_res); a.w.resize(4 * (size_t)new_res);
    for (int i = 0; i < new_res; ++i) {
        const float center = ((float)i + 0.5f) * (float)old_res / (float)new_res;
        a.first[i] = f2i_sat(floorf((center - 2.0f) + 0.5f));
        float* w = &a.w[4 * (size_t)i];
        for (int j = 0; j < 4; ++j) w[j] = lanczos_w((((float)a.first[i] + (float)j + 0.5f) - center) / 2.0f, 2.0f);
        const float inv = 1.0f / (w[0] + w[1] + w[2] + w[3]);
        for (int j = 0; j < 4; ++j) w[j] *= inv;
    }
    return a;
}
static int wrap_repeat(int a, int n) { int r = a - (a / n) * n; return r < 0 ? r + n : r; }
static int wrap_index(uint32_t wrap, int a, int n) {  // the match in MipMap::new's resampling loops (mipmap.rs:88-92): Black leaves the index alone
    if (wrap == PBRT_WRAP_REPEAT) return wrap_repeat(a, n);
    if (wrap == PBRT_WRAP_CLAMP) return std::min(std::max(a, 0), n - 1);
    return a;
}
// MipMap::new (mipmap.rs:60-196): Lanczos zoom to the next power of two where needed, then the box-filtered pyramid.
static void build_pyramid(const float* rgb_in, int w, int h, uint32_t wrap, std::vector<MipLevel>& pyr) {
    std::vector<float> resampled;
    const float* rgb = rgb_in;
    if ((w & (w - 1)) || (h & (h - 1))) {  // mipmap.rs:65-149: zoom in s, then in t, clamp to >= 0
        auto pow2_ceil = [](int v) { int r = 1; while (r < v) r <<= 1; return r; };  // round_up_pow2_32
        const int pw = pow2_ceil(w), ph = pow2_ceil(h);
        std::vector<Sp> tmp((size_t)pw * ph, sp1(0.0f));
        const AxisResample sx = resample_axis(w, pw);
        for (int t = 0; t < h; ++t)
            for (int s = 0; s < pw; ++s) {
                Sp acc = sp1(0.0f);
                for (int j = 0; j < 4; ++j) {
                    const int os = wrap_index(wrap, sx.first[s] + j, w);
                    if (os < 0 || os >= w) continue;
                    const float* px = rgb_in + 3 * ((size_t)t * w + os);
                    acc = acc + mksp(px[0], px[1], px[2]) * sx.w[4 * (size_t)s + j];
                }
                tmp[(size_t)t * pw + s] = acc;
            }
        const AxisResample sy = resample_axis(h, ph);
        std::vector<Sp> col(ph);
        for (int s = 0; s < pw; ++s) {
            for (int t = 0; t < ph; ++t) {
                Sp acc = sp1(0.0f);
                for (int j = 0; j < 4; ++j) {
                    const int ot = wrap_index(wrap, sy.first[t] + j, h);
                    if (ot < 0 || ot >= h) continue;
                    acc = acc + tmp[(size_t)ot * pw + s] * sy.w[4 * (size_t)t + j];
                }
                col[t] = acc;
            }
            for (int t = 0; t < ph; ++t) tmp[(size_t)t * pw + s] = mksp(clampf(col[t].r, 0.0f, INFINITY), clampf(col[t].g, 0.0f, INFINITY), clampf(col[t].b, 0.0f, INFINITY));
        }
        resampled.resize(3 * (size_t)pw * ph);
        for (size_t i = 0; i < (size_t)pw * ph; ++i) { resampled[3 * i] = tmp[i].r; resampled[3 * i + 1] = tmp[i].g; resampled[3 * i + 2] = tmp[i].b; }
        rgb = resampled.data();
        w = pw; h = ph;
    }
    pyr.clear();
    pyr.push_back(MipLevel{w, h, std::vector<Sp>((size_t)w * h), wrap});
    for (size_t i = 0; i < (size_t)w * h; ++i) pyr[0].t[i] = mksp(rgb[3 * i], rgb[3 * i + 1], rgb[3 * i + 2]);
    const size_t n_levels = 1 + (size_t)f2i_sat(log2f((float)std::max(w, h)));
    for (size_t i = 1; i < n_levels; ++i) {
        const MipLevel& f = pyr[i - 1];
        MipLevel c{std::max(1, f.us / 2), std::max(1, f.vs / 2), {}, wrap};
        c.t.resize((size_t)c.us * c.vs);
        for (int t = 0; t < c.vs; ++t)
            for (int s = 0; s < c.us; ++s)
                c.t[(size_t)t * c.us + s] = (mip_texel(f, 2 * s, 2 * t) + mip_texel(f, 2 * s + 1, 2 * t) + mip_texel(f, 2 * s, 2 * t + 1) + mip_texel(f, 2 * s + 1, 2 * t + 1)) * 0.25f;
        pyr.push_back(std::move(c));
    }
}
static void build_env(const float* rgb_in, int w, int h, HostEnv& e) {
    std::vector<MipLevel> pyr;
    build_pyramid(rgb_in, w, h, PBRT_WRAP_REPEAT, pyr);
    w = pyr[0].us; h = pyr[0].vs;
    e.w = w; e.h = h;
    e.texels.resize((size_t)w * h);
    for (size_t i = 0; i < (size_t)w * h; ++i) e.texels[i] = make_float4(pyr[0].t[i].r, pyr[0].t[i].g, pyr[0].t[i].b, 0.0f);
    e.power_L = mip_lookup(pyr, 0.5f, 0.5f, 0.5f);
    const int nu = 2 * w, nv = 2 * h;
    e.nu = nu; e.nv = nv;
    const float fwidth = 0.5f / fminf((float)nu, (float)nv);
    e.cond_func.resize((size_t)nu * nv);
    e.cond_cdf.resize((size_t)(nu + 1) * nv);
    e.cond_int.resize(nv);
    e.marg_func.resize(nv);
    std::vector<float> row(nu), cdf;
    for (int v = 0; v < nv; ++v) {
        const float vp = ((float)v + 0.5f) / (float)nv;
        const float sin_theta = sinf(PB_PI * ((float)v + 0.5f) / (float)nv);
        for (int u = 0; u < nu; ++u) {
            const float up = ((float)u + 0.5f) / (float)nu;
            row[u] = lum(mip_lookup(pyr, up, vp, fwidth)) * sin_theta;
        }
        float fi;
        make_distribution(row, cdf, fi);
        std::copy(row.begin(), row.end(), e.cond_func.begin() + (size_t)v * nu);
        std::copy(cdf.begin(), cdf.end(), e.cond_cdf.begin() + (size_t)v * (nu + 1));
        e.cond_int[v] = fi;
        e.marg_func[v] = fi;
    }
    make_distribution(e.marg_func, e.marg_cdf, e.marg_int);
}
// HaltonSampler tables (samplers/halton.rs:18-26, lowdiscrepancy.rs:18-147,2165-2187, rng.rs, sampling.rs:202-212): the first
// 1000 primes, their prefix sums, and RADICAL_INVERSE_PERMUTATIONS -- each prime's digits shuffled with PCG32's default
// stream, prime after prime, so the whole table is one deterministic constant of the reference.
struct HaltonTables {
    std::vector<uint4> dims;      // {prime, prefix sum, lo, hi of ceil(2^64 / prime)}
    std::vector<uint16_t> perms;
    HaltonTables() {
        std::vector<uint32_t> primes;
        for (uint32_t c = 2; primes.size() < 1000; ++c) {
            bool is_prime = true;
            for (uint32_t q : primes) { if (q * q > c) break; if (c % q == 0) { is_prime = false; break; } }
            if (is_prime) primes.push_back(c);
        }
        uint64_t state = 0x853c49e6748fea9bULL;
        const uint64_t inc = 0xda3e39cb94b95bdbULL;
        auto next_u32 = [&]() -> uint32_t {
            uint64_t old = state;
            state = old * 0x5851f42d4c957f2dULL + inc;
            uint32_t xorshifted = (uint32_t)(((old >> 18) ^ old) >> 27), rot = (uint32_t)(old >> 59);
            return (xorshifted >> rot) | (xorshifted << ((~rot + 1u) & 31));
        };
        uint32_t sum = 0;
        for (uint32_t pr : primes) {
            const unsigned __int128 one = (unsigned __int128)1 << 64;
            const uint64_t magic = (uint64_t)((one + pr - 1) / pr);
            dims.push_back(make_uint4(pr, sum, (uint32_t)magic, (uint32_t)(magic >> 32)));
            const size_t p0 = perms.size();
            for (uint32_t j = 0; j < pr; ++j) perms.push_back((uint16_t)j);
            for (uint32_t k = 0; k < pr; ++k) {  // shuffle(.., count = prime, n_dimensions = 1, rng)
                const uint32_t b = pr - k, threshold = (~b + 1u) & b;  // rng.rs:61 as written (`&`)
                uint32_t r;
                do { r = next_u32(); } while (r < threshold);
                std::swap(perms[p0 + k], perms[p0 + k + r % b]);
            }
            sum += pr;
        }
    }
};
static const HaltonTables& halton_tables() { static HaltonTables t; return t; }
static uint64_t halton_mult_inverse(int64_t a, int64_t n) {  // halton.rs:32-52
    std::function<void(uint64_t, uint64_t, int64_t&, int64_t&)> egcd = [&](uint64_t x, uint64_t y, int64_t& u, int64_t& v) {
        if (y == 0) { u = 1; v = 0; return; }
        int64_t d = (int64_t)x / (int64_t)y, up = 0, vp = 0;
        egcd(y, x % y, up, vp);
        u = vp;
        v = up - d * vp;
    };
    int64_t x = 0, y = 0;
    egcd((uint64_t)a, (uint64_t)n, x, y);
    int64_t r = x - (x / n) * n;
    if (r < 0) r += n;
    return (uint64_t)r;
}
// radical_inverse on the host for the 128 x 5 Halton points of the light grid (lowdiscrepancy.rs:1080-1145)
float host_radical_inverse(int base_index, uint64_t a) {
    static const uint64_t primes[5] = {2, 3, 5, 7, 11};
    if (base_index == 0) {
        uint64_t r = 0;
        for (int i = 0; i < 64; ++i) if (a & (1ull << i)) r |= 1ull << (63 - i);
        return (float)r * 5.421010862427522e-20f;
    }
    const uint64_t base = primes[base_index];
    const float inv_base = 1.0f / (float)base;
    uint64_t reversed = 0;
    float inv_base_n = 1.0f;
    while (a != 0) {
        uint64_t next = a / base, digit = a - next * base;
        reversed = reversed * base + digit;
        inv_base_n *= inv_base;
        a = next;
    }
    return fminf((float)reversed * inv_base_n, PB_ONE_MINUS_EPSILON);
}
int round_up_pow2_32(int v) { v--; v |= v >> 1; v |= v >> 2; v |= v >> 4; v |= v >> 8; v |= v >> 16; return v + 1; }

}  // namespace

// Per-device render scratch (wavefront state, queues, light-grid tables).  It is owned by the library, not by a
// scene, so that re-creating a scene (the end-to-end path uploads it every step) does not re-allocate gigabytes;
// only the allocation is kept, every render rebuilds the contents.  One render at a time per device (mutex).
struct BatchCtx {
    DevBuf<float4> f4[9], rays, rays_pre;
    DevBuf<float4> rec[3];                          // path integrator: the interleaved state records A / B / C (DPaths)
    DevBuf<uint32_t> ray_keys, ray_perm, ray_hist;  // coherence order of the ray queue (k_ray_*)
    DevBuf<float> ao_weight;                        // AOIntegrator: dot(wi, n) / (pdf n) per any-hit ray
    DevBuf<uint32_t> hit_inst, mis_inst;            // instanced scenes: instance of the path / MIS hit
    DevBuf<float4> ray_diff;                        // textured scenes: camera-ray differentials (k_raygen -> k_texture)
    DevBuf<DMaterial> slot_mat;                     // textured scenes: per-slot lobe lists (k_texture -> k_shade)
    DevBuf<float4> slot_frame;                      // and bump-mapped shading frames
    DevBuf<uint32_t> occl, cls_queue, queue[2], counts, dim;
    DevBuf<uint2> sobol;
    DevBuf<float2> pfilm;
    DevBuf<int> g_state;
    DevBuf<float> g_func, g_cdf, g_fint, g_contrib;
    DevBuf<uint32_t> g_request;
    DevBuf<int> g_row;
    cudaStream_t stream = nullptr;
};
struct DirectBufs { DevBuf<uint32_t> u32; DevBuf<float4> f4; };
struct DeviceScratch {
    BatchCtx ctx[4];
    DevBuf<float> filter_table;
    DevBuf<uint4> h_dims;           // HaltonSampler tables, uploaded on first use
    DevBuf<uint16_t> h_perm;
    DevBuf<uint32_t> nibT;          // per-render transposed Sobol' nibble tables for k_shade
    DevBuf<uint32_t> tiles;         // tile-interleaved renders: this share's tile list
    DirectBufs direct;              // DirectLighting / Whitted state (pb_direct.cuh)
    std::vector<uint32_t> h_nibT;
    // timing events are pooled per device: a frame records four per wavefront iteration, and cudaEventCreate / Destroy of several
    // hundred events was a measurable part of the fixed cost of a render call
    // pbrt_gpu_scene_create: pinned staging for the flattened triangle records (written by the host threads, DMA'd from there while
    // the next chunk is being flattened) and the two upload streams; stage_mu serialises scene creation per device
    unsigned char* stage = nullptr;
    size_t stage_n = 0;
    cudaStream_t up_stream[2] = {nullptr, nullptr};
    cudaEvent_t slot_ev[2] = {nullptr, nullptr};
    std::mutex stage_mu;
    bool pool_ready = false;
    cudaError_t staging(size_t bytes) {
        if (stage && stage_n >= bytes) return cudaSuccess;
        if (stage) cudaFreeHost(stage);
        stage = nullptr; stage_n = 0;
        cudaError_t e = cudaHostAlloc((void**)&stage, bytes, cudaHostAllocDefault);
        if (e == cudaSuccess) stage_n = bytes;
        return e;
    }
    // the film of the host-buffer entry points (pbrt_gpu_render, pbrt_gpu_render_multi) and its pinned host mirror live here too, so
    // that a caller who re-creates the scene for every frame does not re-allocate them; film_mu serialises those entry points per device
    DevBuf<float> film;
    float* h_film = nullptr;
    size_t h_film_n = 0;
    std::mutex film_mu;
    cudaError_t host_film(size_t n) {
        if (h_film && h_film_n >= n) return cudaSuccess;
        if (h_film) cudaFreeHost(h_film);
        h_film = nullptr; h_film_n = 0;
        cudaError_t e = cudaHostAlloc((void**)&h_film, n * sizeof(float), cudaHostAllocDefault);
        if (e == cudaSuccess) h_film_n = n;
        return e;
    }
    // loops whose length is only known on the device (null-surface paths, the DirectLighting / Whitted recursion) read their "work
    // left" word through these pinned slots one iteration late, so the device always has the next iteration queued
    uint32_t* h_poll = nullptr;
    cudaError_t poll_words(uint32_t** p) {
        if (!h_poll) {
            cudaError_t e = cudaHostAlloc((void**)&h_poll, 16 * sizeof(uint32_t), cudaHostAllocDefault);
            if (e != cudaSuccess) return e;
        }
        *p = h_poll;
        return cudaSuccess;
    }
    std::vector<cudaEvent_t> ev_pool;
    size_t ev_used = 0;
    cudaError_t event(cudaEvent_t* e) {
        if (ev_used == ev_pool.size()) {
            cudaEvent_t n;
            cudaError_t rc = cudaEventCreate(&n);
            if (rc != cudaSuccess) return rc;
            ev_pool.push_back(n);
        }
        *e = ev_pool[ev_used++];
        return cudaSuccess;
    }
    std::mutex mu;
};
// bytes one stream context may spend on the spatial light distribution's voxel tables before they go sparse
static size_t lightgrid_budget() {
    if (const char* e = std::getenv("PB_LIGHTGRID_BYTES")) {
        const long long v = std::atoll(e);
        if (v > 0) return (size_t)v;
    }
    return (size_t)4 << 30;
}
static DeviceScratch* scratch_for(int device) {
    static DeviceScratch* pool[64] = {nullptr};
    static std::mutex pool_mu;
    std::lock_guard<std::mutex> g(pool_mu);
    if (device < 0 || device >= 64) return nullptr;
    if (!pool[device]) pool[device] = new DeviceScratch();  // lives until process exit
    return pool[device];
}

struct PbrtScene {
    int device = 0;
    DScene d;
    DevBuf<float4> nodes, tri_verts, wide;
    DevBuf<uint4> tri_idx;
    DevBuf<float> vn, vuv, vs;
    DevBuf<DMaterial> materials, materials_single;  // the second list: allow_multiple_lobes = false (Direct / Whitted integrators)
    DevBuf<DLight> lights;
    DevBuf<uint32_t> m32, nib;
    DevBuf<uint64_t> vdc, vdci;
    DevBuf<float> halton;
    std::vector<DLight> h_lights;
    std::vector<uint32_t> h_nib;
    struct EnvBufs { DevBuf<float4> texels; DevBuf<float> cond_func, cond_cdf, cond_int, marg_func, marg_cdf; };
    std::vector<std::unique_ptr<EnvBufs>> env_bufs;
    DevBuf<DEnv> envs;
    DevBuf<DInstance> instances;
    DevBuf<uint2> mesh_alpha;
    std::vector<std::unique_ptr<DevBuf<float4>>> tex_bufs;  // image textures: one pyramid each
    DevBuf<DTexture> textures;
    DevBuf<DMatSrc> mat_src;
    DevBuf<float> ewa_lut;
    std::vector<Sp> h_env_power;  // per light: lmap.lookup((.5,.5), .5) for InfiniteAreaLight::power
    bool has_null_material = false;
    bool cam_motion = false;  // the camera is animated: k_raygen<true> interpolates cam_mo at each sample's time
    DMotion cam_mo;
    bool area_only = true;  // every light is a DiffuseAreaLight: k_shade<true> has the other kinds compiled out
    uint32_t class_mask = 0;  // bit c: some material has shading class c (1..8: a single lobe of kind c - 1; 9: Lambert + microfacet reflection; 10..15: everything else)
    size_t upload_bytes = 0;
    DevBuf<DCounters> counters;
    DevBuf<float> film, samples;
    size_t capacity = 0;
    void recycle_buffers(int dev) {  // every allocation that lives and dies with the scene goes through the device's BufCache
        nodes.cache_dev = tri_verts.cache_dev = wide.cache_dev = tri_idx.cache_dev = vn.cache_dev = vuv.cache_dev = vs.cache_dev = dev;
        materials.cache_dev = materials_single.cache_dev = lights.cache_dev = m32.cache_dev = nib.cache_dev = vdc.cache_dev = vdci.cache_dev = halton.cache_dev = dev;
        envs.cache_dev = instances.cache_dev = mesh_alpha.cache_dev = textures.cache_dev = mat_src.cache_dev = ewa_lut.cache_dev = counters.cache_dev = dev;
    }
};

// The k_trace<COUNT, 0, SMEM, INST> variant a render uses, and its persistent grid: object instances take the two-level traversal
// over global memory, a scene of at most PB_TRACE_SMEM_BYTES is staged in shared memory, anything else walks global memory.
// PB_WIDE=0: A/B switch back to the reference-layout traversal for the scenes that have wide records.  (A plain function on purpose:
// a static local of an inline member function is a GNU-unique symbol, shared by every copy of the library a process loads, which
// made the A/B harness compare a build with itself.)
static bool wide_enabled() {
    static const bool on = !(getenv("PB_WIDE") && atoi(getenv("PB_WIDE")) == 0);
    return on;
}
// PB_WIDE_SPEC=1: the wide traversal with one leaf of look-ahead per lane (pb_trace.cuh::trace_rays_wide_spec; scenes without instances)
static bool wide_spec_enabled() {
    static const bool on = getenv("PB_WIDE_SPEC") && atoi(getenv("PB_WIDE_SPEC")) != 0;
    return on;
}
struct TraceLauncher {
    bool count_work = false, inst = false, smem = false, alpha = false, wide = false, wide_spec = false;
    int wide_walk = 16;
    size_t smem_bytes = 0;
    int grid = 1, blocks_per_sm = 1;
    // one switch over the instantiations the render paths use (MODE 0): F is called with the kernel's address
    template <typename F> void with_kernel(F&& f) const {
        if (alpha) {
            if (inst) { if (count_work) f(k_trace<true, 0, false, true, true>); else f(k_trace<false, 0, false, true, true>); }
            else { if (count_work) f(k_trace<true, 0, false, false, true>); else f(k_trace<false, 0, false, false, true>); }
        } else if (inst) { if (count_work) f(k_trace<true, 0, false, true>); else f(k_trace<false, 0, false, true>); }
        else if (smem) { if (count_work) f(k_trace<true, 0, true>); else f(k_trace<false, 0, true>); }
        else { if (count_work) f(k_trace<true, 0, false>); else f(k_trace<false, 0, false>); }
    }
    cudaError_t init(const PbrtScene* sc, bool count, int sm_count) {
        count_work = count;
        inst = sc->d.n_instances > 0;
        alpha = sc->d.mesh_alpha != nullptr;
        const size_t scene_bytes = (size_t)sc->d.n_nodes * 32 + (size_t)sc->d.n_tris * 48;
        smem = !inst && !alpha && scene_bytes > 0 && scene_bytes <= PB_TRACE_SMEM_BYTES;
        smem_bytes = smem ? scene_bytes : 0;
        wide = wide_enabled() && sc->d.wide != nullptr && !count_work && !alpha && !smem;
        // record visits per lane and round before the warp re-synchronises: long walks keep the lanes that already hold a leaf waiting,
        // which costs more the longer a record fetch takes -- 6 when the records do not fit in L2 (the 4.3 M-triangle statue), 16 when
        // they do (the conference scene); PB_WIDE_WALK overrides
        {
            int l2 = 0;
            cudaDeviceGetAttribute(&l2, cudaDevAttrL2CacheSize, sc->device);
            wide_walk = (size_t)sc->d.n_nodes * 64 > (size_t)std::max(l2, 1) ? 6 : 16;
            if (const char* e_ = getenv("PB_WIDE_WALK")) wide_walk = std::min(64, std::max(1, atoi(e_)));
        }
        int bps = 1;
        cudaError_t e = cudaSuccess;
        wide_spec = wide && !inst && wide_spec_enabled();
        if (wide_spec) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, k_trace_wide_spec, PB_TRACE_THREADS, 0);
        else if (wide) e = inst ? cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, k_trace_wide_inst, PB_TRACE_THREADS, 0)
                           : cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, k_trace_wide_plain, PB_TRACE_THREADS, 0);
        else with_kernel([&](auto k) { e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, k, PB_TRACE_THREADS, smem_bytes); });
        blocks_per_sm = bps;
        grid = sm_count * std::max(1, bps);
        return e;
    }
    void launch(const DScene& d, const TraceIO& io, const uint32_t* d_nrays, uint32_t* d_cursor, DCounters* cnt, cudaStream_t s) const {
        if (wide_spec) k_trace_wide_spec<<<grid, PB_TRACE_THREADS, 0, s>>>(d, io, d_nrays, d_cursor, cnt, wide_walk);
        else if (wide) {
            if (inst) k_trace_wide_inst<<<grid, PB_TRACE_THREADS, 0, s>>>(d, io, d_nrays, d_cursor, cnt, wide_walk);
            else k_trace_wide_plain<<<grid, PB_TRACE_THREADS, 0, s>>>(d, io, d_nrays, d_cursor, cnt, wide_walk);
        } else if (alpha) {
            if (inst) { if (count_work) k_trace<true, 0, false, true, true><<<grid, PB_TRACE_THREADS, 0, s>>>(d, io, d_nrays, 0, d_cursor, cnt); else k_trace<false, 0, false, true, true><<<grid, PB_TRACE_THREADS, 0, s>>>(d, io, d_nrays, 0, d_cursor, cnt); }
            else { if (count_work) k_trace<true, 0, false, false, true><<<grid, PB_TRACE_THREADS, 0, s>>>(d, io, d_nrays, 0, d_cursor, cnt); else k_trace<false, 0, false, false, true><<<grid, PB_TRACE_THREADS, 0, s>>>(d, io, d_nrays, 0, d_cursor, cnt); }
        } else if (inst) {
            if (count_work) k_trace<true, 0, false, true><<<grid, PB_TRACE_THREADS, 0, s>>>(d, io, d_nrays, 0, d_cursor, cnt);
            else k_trace<false, 0, false, true><<<grid, PB_TRACE_THREADS, 0, s>>>(d, io, d_nrays, 0, d_cursor, cnt);
        } else if (smem) {
            if (count_work) k_trace<true, 0, true><<<grid, PB_TRACE_THREADS, smem_bytes, s>>>(d, io, d_nrays, 0, d_cursor, cnt);
            else k_trace<false, 0, true><<<grid, PB_TRACE_THREADS, smem_bytes, s>>>(d, io, d_nrays, 0, d_cursor, cnt);
        } else {
            if (count_work) k_trace<true, 0, false><<<grid, PB_TRACE_THREADS, 0, s>>>(d, io, d_nrays, 0, d_cursor, cnt);
            else k_trace<false, 0, false><<<grid, PB_TRACE_THREADS, 0, s>>>(d, io, d_nrays, 0, d_cursor, cnt);
        }
    }
};

// Host threads this process may use for scene creation: the affinity mask, capped by the cgroup CPU quota (a container that shows 128
// logical CPUs may be allowed 16), shared between the ranks of a one-process-per-GPU launch (LOCAL_WORLD_SIZE), at most 32.
static unsigned host_threads() {
    static const unsigned n = [] {
        unsigned c = std::max(1u, std::thread::hardware_concurrency());
        cpu_set_t set;
        if (sched_getaffinity(0, sizeof set, &set) == 0) c = std::max(1, CPU_COUNT(&set));
        if (FILE* f = fopen("/sys/fs/cgroup/cpu.max", "r")) {
            char quota[32] = {0};
            long period = 0;
            if (fscanf(f, "%31s %ld", quota, &period) == 2 && strcmp(quota, "max") != 0 && period > 0) c = std::min<unsigned>(c, (unsigned)std::max(1L, (atol(quota) + period / 2) / period));
            fclose(f);
        }
        if (const char* w = getenv("LOCAL_WORLD_SIZE")) c = std::max(1u, c / (unsigned)std::max(1, atoi(w)));
        return std::min(32u, c);
    }();
    return n;
}

static int check_device(int device) {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) return fail(PBRT_E_NO_DEVICE, "no CUDA device: the GPU path has no CPU fallback");
    if (device < 0 || device >= n) return fail(PBRT_E_INVALID, "device ordinal out of range");
    // (checked once per device: cudaGetDeviceProperties is a slow call that queues behind every other user of the driver, and it
    // stalled scene_create on a shared host)
    static std::atomic<int> ok[64];
    if (device >= 64 || ok[device].load() == 0) {
        int major = 0, minor = 0;
        CK(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device));
        CK(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, device));
        // sm_90a code loads on compute capability 9.0 and nothing else
        if (major != 9 || minor != 0) return fail(PBRT_E_NO_DEVICE, "kernels are built for sm_90a (H100) only");
        if (device < 64) ok[device].store(1);
    }
    CK(cudaSetDevice(device));
    return PBRT_OK;
}

// SMs of `device` (132 on an H100 SXM): persistent grids and grid-stride launches are sized from it
static int sm_count_of(int device) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || n <= 0) n = 132;
    return n;
}

extern "C" {

const char* pbrt_gpu_last_error(void) { return g_err.c_str(); }
int pbrt_gpu_abi_version(void) { return PBRT_GPU_ABI_VERSION; }
uint64_t pbrt_gpu_launch_count(void) { return g_launches.load(); }

int pbrt_gpu_scene_create(const PbrtSceneDesc* desc, int device, PbrtScene** out) {
    if (!desc || !out) return fail(PBRT_E_INVALID, "null argument");
    static const int timing = getenv("PB_TIMING") ? atoi(getenv("PB_TIMING")) : 0;  // 1: every call; 2: only calls slower than 100 ms
    const auto t_enter = std::chrono::steady_clock::now();
    std::string timing_log;
    auto since = [&](const char* what) {
        if (!timing) return;
        char line[160];
        snprintf(line, sizeof line, "[pb timing] scene_create %-26s %8.3f ms\n", what, std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_enter).count());
        if (timing == 1) fputs(line, stderr); else timing_log += line;
    };
    struct SlowDump { std::string& log; const std::chrono::steady_clock::time_point t0; int mode; ~SlowDump() {
        if (mode == 2 && std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count() > 100.0) fputs(log.c_str(), stderr); } } slow_dump{timing_log, t_enter, timing};
    *out = nullptr;
    if ((desc->n_nodes && !desc->nodes) || (desc->n_tris && !desc->tris) || (desc->n_meshes && !desc->meshes) ||
        (desc->n_materials && !desc->materials) || (desc->n_lights && !desc->lights))
        return fail(PBRT_E_INVALID, "null array in scene description");
    // ---- validate + flatten on the host ------------------------------------------------------
    std::vector<size_t> vbase(desc->n_meshes + 1, 0);
    bool any_n = false, any_uv = false, any_s = false, any_alpha = false;
    for (uint32_t i = 0; i < desc->n_meshes; ++i) {
        const PbrtMesh& m = desc->meshes[i];
        if (!m.p) return fail(PBRT_E_INVALID, "mesh without positions");
        for (uint32_t a : {m.alpha, m.shadow_alpha}) {  // TriangleMesh.alpha_mask / shadow_alpha_mask: float textures
            if (!a) continue;
            if (a > desc->n_textures || !desc->textures) return fail(PBRT_E_INVALID, "alpha mask texture index out of range");
            if (desc->textures[a - 1].channels != 1) return fail(PBRT_E_INVALID, "an alpha mask is a float texture");
            any_alpha = true;
        }
        vbase[i + 1] = vbase[i] + m.n_verts;
        any_n |= m.n != nullptr; any_uv |= m.uv != nullptr; any_s |= m.s != nullptr;
    }
    const size_t total_verts = vbase[desc->n_meshes];
    std::vector<DMaterial> mats(desc->n_materials);
    std::vector<DMaterial> mats_single(desc->n_materials);  // the lobe lists without allow_multiple_lobes (DirectLighting / Whitted: directlighting.rs:77)
    for (uint32_t i = 0; i < desc->n_materials; ++i) {
        const char* why = "";
        if (!compile_material_at(desc->materials, desc->n_materials, i, mats[i], true, nullptr, &why) ||
            !compile_material_at(desc->materials, desc->n_materials, i, mats_single[i], false, nullptr, &why))
            return fail(std::strstr(why, "child index") ? PBRT_E_INVALID : PBRT_E_UNSUPPORTED, why);
    }
    {  // shading classes: materials with the same lobe-kind / Fresnel-kind sequence run the same code path.  Classes 1..8 are exactly "one
       // lobe of kind class - 1" (what k_shade<.., SPEC = class> is compiled for; a textured material leaves them again below, because its
       // lobe list can change from hit to hit); class 9 is "Lambert, then microfacet reflection" (plastic; k_shade<.., PB_SPEC_PLASTIC>);
       // classes 10..15 hold everything else and may share a class between signatures.
        const int first_general = PB_SPEC_PLASTIC + 1;  // 10
        std::vector<uint64_t> sigs;
        for (DMaterial& m : mats) {
            bool scaled = false;  // a MixMaterial's lobes carry sc_opt, which only the general instantiation reads
            for (int k = 0; k < m.n_lobes; ++k) scaled = scaled || m.lobes[k].has_sc != 0;
            if (!scaled && m.n_lobes == 1 && m.lobes[0].kind <= LOBE_FRESNEL_BLEND) { m.cls = 1 + m.lobes[0].kind; continue; }
            if (!scaled && m.n_lobes == 2 && m.lobes[0].kind == LOBE_LAMBERT && m.lobes[1].kind == LOBE_MF_REFL) { m.cls = PB_SPEC_PLASTIC; continue; }
            uint64_t sig = 1;
            for (int k = 0; k < m.n_lobes; ++k) sig = sig * 128 + (uint64_t)(m.lobes[k].kind * 8 + m.lobes[k].fresnel * 2 + (m.lobes[k].has_sc ? 1 : 0)) + 1;
            size_t j = 0;
            while (j < sigs.size() && sigs[j] != sig) ++j;
            if (j == sigs.size()) sigs.push_back(sig);
            m.cls = first_general + (int)(j % (PB_SHADE_CLASSES - first_general));
        }
    }
    // image textures (ABI v3): the class above is that of the all-constants lobe list; what k_shade runs on comes from k_texture
    if (desc->n_textures && !desc->textures) return fail(PBRT_E_INVALID, "null texture array");
    std::vector<DMatSrc> mat_src(desc->n_textures ? desc->n_materials : 0);
    for (uint32_t i = 0; i < desc->n_materials; ++i) {
        const PbrtMaterial& pm = desc->materials[i];
        bool textured = false;
        if (pm.bump) {
            if (pm.bump > desc->n_textures) return fail(PBRT_E_INVALID, "bump map texture index out of range");
            if (desc->textures[pm.bump - 1].channels != 1) return fail(PBRT_E_INVALID, "a bump map is a float texture");
            textured = true;
        }
        for (int g = 0; g < PBRT_MAX_TEX_GROUPS; ++g) {
            if (!pm.tex[g]) continue;
            if (pm.tex[g] > desc->n_textures) return fail(PBRT_E_INVALID, "material texture index out of range");
            int nv = 0;
            if (pbrt_material_tex_offset(pm.kind, g, &nv) < 0) return fail(PBRT_E_UNSUPPORTED, "texture bound to a parameter group this material kind does not have");
            if ((uint32_t)nv != desc->textures[pm.tex[g] - 1].channels) return fail(PBRT_E_INVALID, "spectrum parameter bound to a float texture or vice versa");
            textured = true;
        }
        if (!desc->n_textures) continue;
        DMatSrc& ms = mat_src[i];
        std::memset(&ms, 0, sizeof ms);
        ms.kind = pm.kind;
        std::memcpy(ms.params, pm.params, sizeof ms.params);
        std::memcpy(ms.tex, pm.tex, sizeof ms.tex);
        material_alphas(pm, ms.alpha_u, ms.alpha_v);
        for (int g = 0; g < PBRT_MAX_TEX_GROUPS; ++g) {
            int nv = 0;
            const int o = pbrt_material_tex_offset(pm.kind, g, &nv);
            ms.tex_off[g] = (uint8_t)(o < 0 ? 0 : o);
            if (o >= 0 && nv == 3) ms.n_spectrum = (uint32_t)g + 1u;
        }
        ms.bump = pm.bump;
        if (textured && mats[i].cls <= PB_SPEC_PLASTIC) mats[i].cls = PB_SHADE_CLASSES - 1;  // not a compile-time lobe list any more
        if (textured) mats[i].cls |= PB_MAT_TEXTURED;
        if (pm.bump) mats[i].cls |= PB_MAT_BUMPED;
    }
    std::vector<int> tex_depth(desc->n_textures, 1);
    for (uint32_t i = 0; i < desc->n_textures; ++i) {
        const PbrtTexture& t = desc->textures[i];
        if (t.channels != 1 && t.channels != 3) return fail(PBRT_E_INVALID, "texture channels must be 1 or 3");
        if (t.kind == PBRT_TEX_IMAGE) {
            if (!t.texels || t.res[0] == 0 || t.res[1] == 0) return fail(PBRT_E_INVALID, "texture without texels");
            if (t.res[0] > 16384 || t.res[1] > 16384) return fail(PBRT_E_UNSUPPORTED, "texture larger than 16384 texels on a side");
            if (t.wrap > PBRT_WRAP_CLAMP) return fail(PBRT_E_INVALID, "unknown texture wrap mode");
            if (t.mapping > PBRT_MAP_PLANAR) return fail(PBRT_E_UNSUPPORTED, "texture mapping outside the GPU path");
        } else if (t.kind <= PBRT_TEX_MIX) {
            const int nc = t.kind == PBRT_TEX_CONSTANT ? 0 : (t.kind == PBRT_TEX_SCALE ? 2 : 3);
            for (int c = 0; c < nc; ++c) {
                if (t.child[c] == 0 || t.child[c] > i) return fail(PBRT_E_INVALID, "texture operand must be an earlier texture");
                if (desc->textures[t.child[c] - 1].channels != (c == 2 ? 1u : t.channels)) return fail(PBRT_E_INVALID, "texture operand of the wrong type");
                tex_depth[i] = std::max(tex_depth[i], 1 + tex_depth[t.child[c] - 1]);
            }
            if (tex_depth[i] > PBRT_MAX_TEXTURE_DEPTH) return fail(PBRT_E_UNSUPPORTED, "texture graph deeper than 4 levels");
        } else return fail(PBRT_E_UNSUPPORTED, "texture kind outside the GPU path");
    }
    if (desc->n_instances && !desc->instances) return fail(PBRT_E_INVALID, "null instance array");
    std::vector<DLight> lights(desc->n_lights);
    uint32_t n_inf = 0, inf_idx[PBRT_MAX_INFINITE_LIGHTS] = {0, 0, 0, 0};
    for (uint32_t i = 0; i < desc->n_lights; ++i) {
        const PbrtLight& l = desc->lights[i];
        if (l.kind > PBRT_LIGHT_INFINITE) return fail(PBRT_E_UNSUPPORTED, "light kind outside the GPU path");
        if (l.kind == PBRT_LIGHT_DIFFUSE_AREA && l.tri >= desc->n_tris) return fail(PBRT_E_INVALID, "light triangle out of range");
        std::memset(&lights[i], 0, sizeof(DLight));
        lights[i].kind = l.kind;
        lights[i].L[0] = l.L[0]; lights[i].L[1] = l.L[1]; lights[i].L[2] = l.L[2];
        lights[i].tri = l.tri;
        lights[i].two_sided = l.two_sided ? 1u : 0u;
        for (int k = 0; k < 3; ++k) lights[i].p[k] = l.p[k];
        for (int k = 0; k < 9; ++k) lights[i].w2l[k] = l.w2l[k];
        lights[i].cos_total_width = l.cos_total_width;
        lights[i].cos_falloff_start = l.cos_falloff_start;
        lights[i].area = l.area;
        lights[i].n_samples = l.n_samples ? l.n_samples : 1u;
        if (l.kind == PBRT_LIGHT_INFINITE) {
            const uint32_t w = l.env_res[0], h = l.env_res[1];
            if (!l.env_texels || w == 0 || h == 0) return fail(PBRT_E_INVALID, "infinite light without texels");
            if (w > 16384 || h > 16384) return fail(PBRT_E_UNSUPPORTED, "environment map larger than 16384 texels on a side");
            if (n_inf == PBRT_MAX_INFINITE_LIGHTS) return fail(PBRT_E_UNSUPPORTED, "too many infinite lights");
            inf_idx[n_inf++] = i;
        }
    }
    // The host-side flattening runs on all cores (a 4.3 M-triangle scene is re-uploaded on every end-to-end step).
    const unsigned hw = host_threads();
    auto parallel_for = [&](uint32_t n, const std::function<int(uint32_t, uint32_t)>& body) -> int {
        const unsigned nt = n < 65536 ? 1u : hw;
        std::vector<int> rc(nt, 0);
        std::vector<std::thread> th;
        for (unsigned t = 0; t < nt; ++t) {
            uint32_t lo = (uint32_t)((uint64_t)n * t / nt), hi = (uint32_t)((uint64_t)n * (t + 1) / nt);
            if (nt == 1) rc[0] = body(lo, hi);
            else th.emplace_back([&, t, lo, hi] { rc[t] = body(lo, hi); });
        }
        for (auto& x : th) x.join();
        for (int r : rc) if (r) return r;
        return 0;
    };
    // BVH nodes: PbrtBvhNode already IS the device layout (32 bytes: 6 floats, offset, n_prims | axis << 16 | pad << 24;
    // the kernels mask the pad byte), so the caller's array is validated in place and uploaded without staging.
    static_assert(sizeof(PbrtBvhNode) == 32, "LinearBVHNode layout");
    std::atomic<uint32_t> max_leaf_prims(0);
    int vrc = parallel_for(desc->n_nodes, [&](uint32_t lo, uint32_t hi) -> int {
        uint32_t mx = 0;
        struct Publish { std::atomic<uint32_t>& a; uint32_t& v; ~Publish() { uint32_t c = a.load(); while (v > c && !a.compare_exchange_weak(c, v)) {} } } pub{max_leaf_prims, mx};
        for (uint32_t i = lo; i < hi; ++i) {
            const PbrtBvhNode& n = desc->nodes[i];
            if (n.n_prims > 0) {
                if ((uint64_t)n.offset + n.n_prims > desc->n_tris || n.offset < 0) return 1;
                mx = std::max<uint32_t>(mx, n.n_prims);
            } else if (n.offset <= (int32_t)i || (uint32_t)n.offset >= desc->n_nodes || i + 1 >= desc->n_nodes || n.axis > 2) return 2;
        }
        return 0;
    });
    if (vrc == 1) return fail(PBRT_E_INVALID, "BVH leaf range out of bounds");
    if (vrc == 2) return fail(PBRT_E_INVALID, "BVH interior node malformed");
    since("nodes validated");
    {
        // Tree depth: the traversal stack holds 64 entries like the reference's nodes_to_visit (bvh.rs:420,480), one per interior
        // ancestor whose far child is pending; a deeper tree would index past the reference's array (a panic there) and past the
        // kernel's stack here.  flatten_bvh_tree (bvh.rs:393-400) lays a subtree out as one contiguous block, first child right
        // after its parent, so the tree splits into independent index ranges that are checked on all cores; anything that does not
        // have that layout takes the sequential pass.
        struct Range { uint32_t lo, hi; uint32_t depth; };
        std::vector<Range> work;
        bool layout_ok = true, too_deep = false;
        auto spine_end = [&](uint32_t r) -> uint32_t {  // one past the last node of the subtree rooted at r
            uint32_t i = r;
            for (;;) {
                const PbrtBvhNode& n = desc->nodes[i];
                if (n.n_prims > 0) return i + 1;
                i = (uint32_t)n.offset;
            }
        };
        if (desc->n_nodes) work.push_back({0u, spine_end(0u), 0u});
        for (uint32_t k = 0; k < desc->n_instances && desc->instances; ++k) {
            const uint32_t r = desc->instances[k].root;
            if (r >= desc->n_nodes) return fail(PBRT_E_INVALID, "instance root out of range");
            bool seen = false;
            for (const Range& w : work) seen |= w.lo == r;
            if (!seen) work.push_back({r, spine_end(r), 0u});
        }
        const uint32_t grain = std::max<uint32_t>(4096u, desc->n_nodes / (8u * hw));
        for (size_t k = 0; k < work.size() && layout_ok && !too_deep;) {  // split big ranges at their root
            const Range w = work[k];
            const PbrtBvhNode& n = desc->nodes[w.lo];
            if (w.hi - w.lo <= grain || n.n_prims > 0) { ++k; continue; }
            const uint32_t off = (uint32_t)n.offset;
            if (off <= w.lo + 1 || off >= w.hi) { layout_ok = false; break; }
            if (w.depth >= 64) { too_deep = true; break; }
            work[k] = {w.lo + 1, off, w.depth + 1};
            work.push_back({off, w.hi, w.depth + 1});
        }
        if (layout_ok && !too_deep) {
            std::atomic<size_t> next(0);
            std::atomic<int> bad(0);
            auto run = [&]() {
                std::vector<uint8_t> d;
                for (size_t k = next.fetch_add(1); k < work.size() && !bad.load(); k = next.fetch_add(1)) {
                    const Range w = work[k];
                    d.assign(w.hi - w.lo, 0);
                    d[0] = (uint8_t)w.depth;
                    for (uint32_t i = w.lo; i < w.hi; ++i) {
                        const PbrtBvhNode& n = desc->nodes[i];
                        if (n.n_prims > 0) continue;
                        const uint32_t off = (uint32_t)n.offset;
                        if (i + 1 >= w.hi || off >= w.hi) { bad.store(2); break; }  // not a contiguous subtree after all
                        if (d[i - w.lo] >= 64) { bad.store(1); break; }
                        const uint8_t dch = (uint8_t)(d[i - w.lo] + 1);
                        d[i + 1 - w.lo] = std::max(d[i + 1 - w.lo], dch);
                        d[off - w.lo] = std::max(d[off - w.lo], dch);
                    }
                }
            };
            const unsigned nt = work.size() > 1 ? std::min<unsigned>(hw, (unsigned)work.size()) : 1u;
            std::vector<std::thread> th;
            for (unsigned t = 1; t < nt; ++t) th.emplace_back(run);
            run();
            for (auto& x : th) x.join();
            too_deep = bad.load() == 1;
            layout_ok = bad.load() != 2;
        }
        if (!layout_ok) {  // general forward order (children after their parent is all that was validated): one sequential pass
            too_deep = false;
            std::vector<uint8_t> depth(desc->n_nodes, 0);
            for (uint32_t i = 0; i < desc->n_nodes && !too_deep; ++i) {
                const PbrtBvhNode& n = desc->nodes[i];
                if (n.n_prims > 0) continue;
                if (depth[i] >= 64) { too_deep = true; break; }
                const uint8_t dch = (uint8_t)(depth[i] + 1);
                depth[i + 1] = std::max(depth[i + 1], dch);
                depth[(uint32_t)n.offset] = std::max(depth[(uint32_t)n.offset], dch);
            }
        }
        if (too_deep) return fail(PBRT_E_UNSUPPORTED, "BVH deeper than the 64-entry traversal stack (bvh.rs:420)");
    }
    if (desc->n_instances) {
        // An object's primitives may not be instances themselves (api.rs:3029 rejects ObjectInstance inside ObjectBegin): the two-level
        // traversal keeps ONE current instance, so a nested record would silently report wrong hits.  Walk each distinct object tree.
        if (!desc->instances) return fail(PBRT_E_INVALID, "null instance array");
        std::vector<uint32_t> roots;
        for (uint32_t i = 0; i < desc->n_instances; ++i) {
            if (desc->instances[i].root >= desc->n_nodes) return fail(PBRT_E_INVALID, "instance root out of range");
            roots.push_back(desc->instances[i].root);
        }
        std::sort(roots.begin(), roots.end());
        roots.erase(std::unique(roots.begin(), roots.end()), roots.end());
        std::vector<uint32_t> todo;
        for (uint32_t root : roots) {
            todo.assign(1, root);
            while (!todo.empty()) {
                const uint32_t i = todo.back();
                todo.pop_back();
                const PbrtBvhNode& n = desc->nodes[i];
                if (n.n_prims > 0) {
                    for (uint32_t k = 0; k < n.n_prims; ++k)
                        if (desc->tris[(uint32_t)n.offset + k].mesh == PBRT_MESH_INSTANCE)
                            return fail(PBRT_E_UNSUPPORTED, "an object instance inside an object (nested instancing) is outside the GPU path");
                } else { todo.push_back(i + 1); todo.push_back((uint32_t)n.offset); }
            }
        }
    }
    since("depth + instance checks");
    // ---- device, scene object, and the big uploads ------------------------------------------------------------------------------
    // The caller's arrays go up as they are -- nodes, triangle records, per-vertex attributes -- and the triangles are validated and
    // flattened (pre-gathered vertices in BVH order) by a kernel: the host side of a 4.3 M-triangle scene_create is then the node checks.
    auto tri_error = [&](const PbrtTri& t) -> int {  // what the flattening below rejects
        if (t.mesh == PBRT_MESH_INSTANCE) return t.v[0] >= desc->n_instances ? 5 : 0;
        if (t.mesh >= desc->n_meshes) return 1;
        const PbrtMesh& m = desc->meshes[t.mesh];
        if (t.v[0] >= m.n_verts || t.v[1] >= m.n_verts || t.v[2] >= m.n_verts) return 2;
        if (t.material != PBRT_NO_MATERIAL && t.material >= desc->n_materials) return 3;
        if (t.area_light >= (int32_t)desc->n_lights) return 4;
        if (t.area_light >= 0 && (m.alpha || m.shadow_alpha)) return 6;
        return 0;
    };
    auto tri_fail = [&](int code) -> int {
        if (code == 1) return fail(PBRT_E_INVALID, "triangle mesh index out of range");
        if (code == 2) return fail(PBRT_E_INVALID, "vertex index out of range");
        if (code == 3) return fail(PBRT_E_INVALID, "material index out of range");
        if (code == 4) return fail(PBRT_E_INVALID, "area light index out of range");
        if (code == 6) return fail(PBRT_E_UNSUPPORTED, "alpha mask on an emissive mesh is outside the GPU path (pdf_li would have to evaluate it)");
        return fail(PBRT_E_INVALID, "instance index out of range");
    };
    int rc = check_device(device);
    if (rc != PBRT_OK) {
        // no usable device: a malformed description is still reported as such (validation does not depend on the hardware; it is
        // otherwise fused with the flattening below)
        const std::string dev_err = g_err;
        vrc = parallel_for(desc->n_tris, [&](uint32_t lo, uint32_t hi) -> int {
            for (uint32_t i = lo; i < hi; ++i) if (int e = tri_error(desc->tris[i])) return e;
            return 0;
        });
        if (vrc) return tri_fail(vrc);
        return fail(rc, dev_err);
    }
    DeviceScratch* up_scr = scratch_for(device);
    if (!up_scr) return fail(PBRT_E_INVALID, "device ordinal out of range");
    std::unique_lock<std::mutex> stage_lock(up_scr->stage_mu);
    if (!up_scr->pool_ready) {
        for (int k = 0; k < 2; ++k) CK(cudaStreamCreateWithFlags(&up_scr->up_stream[k], cudaStreamNonBlocking));
        for (int k = 0; k < 2; ++k) CK(cudaEventCreateWithFlags(&up_scr->slot_ev[k], cudaEventDisableTiming));
        up_scr->pool_ready = true;
    }
    std::unique_ptr<PbrtScene> sc_guard(new PbrtScene());
    PbrtScene* sc = sc_guard.get();
    sc->device = device;
    sc->recycle_buffers(device);
    DevBuf<uint2> raw_tris;   // the caller's PbrtTri records as they are (24 B each), flattened on the device
    DevBuf<float> raw_p;      // mesh positions, concatenated
    DevBuf<DMeshRec> d_meshes;
    DevBuf<uint32_t> d_status;
    raw_tris.cache_dev = raw_p.cache_dev = d_meshes.cache_dev = d_status.cache_dev = device;
    CK(sc->nodes.alloc(2 * (size_t)desc->n_nodes));
    CK(sc->tri_verts.alloc(3 * (size_t)desc->n_tris));
    CK(sc->tri_idx.alloc((size_t)desc->n_tris));
    CK(raw_tris.alloc(3 * (size_t)desc->n_tris));
    CK(raw_p.alloc(3 * total_verts));
    if (any_n) CK(sc->vn.alloc(3 * total_verts));
    if (any_uv) CK(sc->vuv.alloc(2 * total_verts));
    if (any_s) CK(sc->vs.alloc(3 * total_verts));
    CK(d_meshes.alloc(std::max<size_t>(desc->n_meshes, 1)));
    CK(d_status.alloc(2));
    since("device buffers allocated");
    // ---- uploads.  A source array in pinned memory (the caller's own cudaHostAlloc / pbrt_gpu_host_register) is DMA'd where it
    // lies; pageable memory goes through two pinned staging slots, copied into them on all cores while the previous slot is in flight
    // (a cudaMemcpy straight from pageable memory runs at a fraction of the pinned rate).
    cudaStream_t ups = up_scr->up_stream[1];
    const size_t slot_bytes = (size_t)64 << 20;
    CK(up_scr->staging(2 * slot_bytes));
    cudaEvent_t* const slot_ev = up_scr->slot_ev;
    bool slot_used[2] = {false, false};
    int next_slot = 0;
    size_t up_bytes = 0;
    auto upload = [&](void* dst, const void* src, size_t bytes) -> cudaError_t {
        if (!bytes) return cudaSuccess;
        up_bytes += bytes;
        cudaPointerAttributes at;
        const bool pinned = cudaPointerGetAttributes(&at, src) == cudaSuccess && at.type == cudaMemoryTypeHost;
        cudaGetLastError();
        if (pinned) return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, ups);
        for (size_t off = 0; off < bytes; off += slot_bytes) {
            const size_t n = std::min(slot_bytes, bytes - off);
            const int k = next_slot;
            next_slot ^= 1;
            if (slot_used[k]) { cudaError_t e = cudaEventSynchronize(slot_ev[k]); if (e != cudaSuccess) return e; }
            unsigned char* stage = up_scr->stage + (size_t)k * slot_bytes;
            const unsigned char* from = static_cast<const unsigned char*>(src) + off;
            if (n < ((size_t)1 << 20)) std::memcpy(stage, from, n);
            else {
                const unsigned nt = hw;
                std::vector<std::thread> th;
                for (unsigned t = 0; t < nt; ++t) th.emplace_back([=] { const size_t lo = n * t / nt, hi = n * (t + 1) / nt; std::memcpy(stage + lo, from + lo, hi - lo); });
                for (auto& x : th) x.join();
            }
            cudaError_t e = cudaMemcpyAsync(static_cast<unsigned char*>(dst) + off, stage, n, cudaMemcpyHostToDevice, ups);
            if (e == cudaSuccess) e = cudaEventRecord(slot_ev[k], ups);
            if (e != cudaSuccess) return e;
            slot_used[k] = true;
        }
        return cudaSuccess;
    };
    std::vector<DMeshRec> h_meshes(std::max<size_t>(desc->n_meshes, 1));
    for (uint32_t i = 0; i < desc->n_meshes; ++i) {
        const PbrtMesh& m = desc->meshes[i];
        uint32_t flags = 0;
        if ((m.reverse_orientation != 0) ^ (m.transform_swaps_handedness != 0)) flags |= TRI_FLIP;
        if (m.n) flags |= TRI_HAS_N;
        if (m.uv) flags |= TRI_HAS_UV;
        if (m.s) flags |= TRI_HAS_S;
        if (m.alpha) flags |= TRI_ALPHA;
        if (m.shadow_alpha) flags |= TRI_SHADOW_ALPHA;
        h_meshes[i].vbase = (uint32_t)vbase[i]; h_meshes[i].n_verts = m.n_verts; h_meshes[i].flags = flags; h_meshes[i].pad = 0;
    }
    if (total_verts >= (1ull << 32)) return fail(PBRT_E_UNSUPPORTED, "more than 2^32 vertices");
    {
        cudaError_t e = cudaMemcpyAsync(d_meshes.p, h_meshes.data(), h_meshes.size() * sizeof(DMeshRec), cudaMemcpyHostToDevice, ups);
        if (e == cudaSuccess) e = cudaMemsetAsync(d_status.p, 0, 8, ups);
        if (e == cudaSuccess) e = upload(raw_tris.p, desc->tris, 24 * (size_t)desc->n_tris);
        for (uint32_t i = 0; i < desc->n_meshes && e == cudaSuccess; ++i) {
            const PbrtMesh& m = desc->meshes[i];
            e = upload(raw_p.p + 3 * vbase[i], m.p, 12 * (size_t)m.n_verts);
        }
        if (e != cudaSuccess) return fail(PBRT_E_CUDA, std::string("upload triangles / positions: ") + cudaGetErrorString(e));
        // triangles: validated and pre-gathered (vertices in BVH order) on the device
        if (desc->n_tris) {
            k_flatten_tris<<<(desc->n_tris + 255) / 256, 256, 0, ups>>>(raw_tris.p, desc->n_tris, d_meshes.p, desc->n_meshes, raw_p.p, desc->n_materials, desc->n_lights,
                                                                       desc->n_instances, sc->tri_verts.p, sc->tri_idx.p, d_status.p);
            g_launches++;
        }
        e = upload(sc->nodes.p, desc->nodes, 32 * (size_t)desc->n_nodes);
        // per-vertex attributes go from the caller's mesh arrays into the concatenated device arrays
        for (uint32_t i = 0; i < desc->n_meshes && e == cudaSuccess; ++i) {
            const PbrtMesh& m = desc->meshes[i];
            if (m.n) e = upload(sc->vn.p + 3 * vbase[i], m.n, 12 * (size_t)m.n_verts);
            if (e == cudaSuccess && m.uv) e = upload(sc->vuv.p + 2 * vbase[i], m.uv, 8 * (size_t)m.n_verts);
            if (e == cudaSuccess && m.s) e = upload(sc->vs.p + 3 * vbase[i], m.s, 12 * (size_t)m.n_verts);
        }
        if (e != cudaSuccess) return fail(PBRT_E_CUDA, std::string("upload nodes / vertex attributes: ") + cudaGetErrorString(e));
    }
    since("uploads queued");
    uint32_t h_status[2] = {0, 0};
    CK(cudaMemcpyAsync(h_status, d_status.p, 8, cudaMemcpyDeviceToHost, ups));
    CK(cudaStreamSynchronize(ups));  // (the staging slots and the temporaries are quiet from here on)
    CK(cudaGetLastError());
    vrc = (int)h_status[0];
    std::atomic<int> null_seen((int)h_status[1]);
    if (vrc) return tri_fail(vrc);
    std::vector<DInstance> dinst(desc->n_instances);
    for (uint32_t i = 0; i < desc->n_instances; ++i) {
        const PbrtInstance& I = desc->instances[i];
        if (I.root >= desc->n_nodes) return fail(PBRT_E_INVALID, "instance root out of range");
        std::memset(&dinst[i], 0, sizeof(DInstance));
        dinst[i].root = I.root;
        dinst[i].identity = I.identity ? 1u : 0u;
        std::memcpy(dinst[i].m, I.m, 64);
        std::memcpy(dinst[i].m_inv, I.m_inv, 64);
    }
    const bool has_null = null_seen.load() != 0;
    since("triangles flattened");
    // ---- Sobol' tables (embedded blob) ---------------------------------------------------------
    const unsigned char* blob = pb_sobol_blob_start;
    size_t blob_size = (size_t)(pb_sobol_blob_end - pb_sobol_blob_start);
    const size_t need = 32 + 1024 * 52 * 4 + (25 + 26) * 52 * 8;
    uint32_t hdr[8];
    if (blob_size < need) return fail(PBRT_E_INVALID, "embedded Sobol table blob truncated");
    std::memcpy(hdr, blob, 32);
    if (hdr[0] != 0x4C424F53u || hdr[1] != 1024 || hdr[2] != 52) return fail(PBRT_E_INVALID, "embedded Sobol table blob corrupt");
    std::vector<uint32_t> m32(1024 * 52);
    std::vector<uint64_t> vdc(25 * 52), vdci(26 * 52);
    std::memcpy(m32.data(), blob + 32, m32.size() * 4);
    std::memcpy(vdc.data(), blob + 32 + m32.size() * 4, vdc.size() * 8);
    std::memcpy(vdci.data(), blob + 32 + m32.size() * 4 + vdc.size() * 8, vdci.size() * 8);
    // nibble tables nib[dim][chunk][e] (pb_sobol.cuh)
    std::vector<uint32_t> nib((size_t)1024 * PB_SOBOL_CHUNKS * 16);
    for (int dim = 0; dim < 1024; ++dim)
        for (int c = 0; c < PB_SOBOL_CHUNKS; ++c)
            for (int e = 0; e < 16; ++e) {
                uint32_t v = 0;
                for (int j = 0; j < 4; ++j)
                    if (e & (1 << j)) v ^= m32[(size_t)dim * 52 + 4 * c + j];
                nib[((size_t)dim * PB_SOBOL_CHUNKS + c) * 16 + e] = v;
            }
    std::vector<float> halton(128 * 5);
    for (int s = 0; s < 128; ++s)
        for (int k = 0; k < 5; ++k) halton[5 * s + k] = host_radical_inverse(k, (uint64_t)s);

    since("tables built");
    sc->has_null_material = has_null;
    sc->h_nib = nib;
    for (const DLight& l : lights) if (l.kind != PBRT_LIGHT_DIFFUSE_AREA) sc->area_only = false;
    for (const DMaterial& m : mats) sc->class_mask |= 1u << (m.cls & 0xff);
    sc->h_lights = lights;
#define UP(buf, vec)                                                                                     \
    do {                                                                                                 \
        cudaError_t e_ = sc->buf.upload(vec);                                                            \
        if (e_ != cudaSuccess) return fail(PBRT_E_CUDA, std::string("upload " #buf ": ") + cudaGetErrorString(e_)); \
        sc->upload_bytes += (vec).size() * sizeof((vec)[0]);                                             \
    } while (0)
    sc->upload_bytes += up_bytes;
    since("nodes + triangles uploaded");
    {   // wide records for the traversal (pb_trace.cuh): derived on the device from the node array that has just arrived
        bool ok = desc->n_nodes > 1 && desc->nodes[0].n_prims == 0 && !any_alpha &&
                  desc->n_nodes < (1u << PB_WIDE_LEAF_SHIFT) && desc->n_tris < (1u << PB_WIDE_LEAF_SHIFT) &&
                  (desc->n_instances > 0 || (size_t)desc->n_nodes * 32 + (size_t)desc->n_tris * 48 > PB_TRACE_SMEM_BYTES) && max_leaf_prims.load() <= 15u;
        if (ok) {
            CK(sc->wide.alloc(4 * (size_t)desc->n_nodes));
            k_wide_build<<<(desc->n_nodes + 255) / 256, 256>>>(sc->nodes.p, desc->n_nodes, sc->wide.p);
            CK(cudaGetLastError());
            g_launches++;
        }
    }
    // infinite lights: radiance map + Distribution2D tables (built on the host like InfiniteAreaLight::new does)
    {
        std::vector<DEnv> envs;
        sc->h_env_power.assign(desc->n_lights, sp1(0.0f));
        for (uint32_t k = 0; k < n_inf; ++k) {
            const PbrtLight& l = desc->lights[inf_idx[k]];
            HostEnv he;
            build_env(l.env_texels, (int)l.env_res[0], (int)l.env_res[1], he);  // he.w / he.h: the power-of-two resolution after MipMap::new's resampling
            sc->env_bufs.emplace_back(new PbrtScene::EnvBufs());
            PbrtScene::EnvBufs& b = *sc->env_bufs.back();
            cudaError_t e_ = b.texels.upload(he.texels);
            if (e_ == cudaSuccess) e_ = b.cond_func.upload(he.cond_func);
            if (e_ == cudaSuccess) e_ = b.cond_cdf.upload(he.cond_cdf);
            if (e_ == cudaSuccess) e_ = b.cond_int.upload(he.cond_int);
            if (e_ == cudaSuccess) e_ = b.marg_func.upload(he.marg_func);
            if (e_ == cudaSuccess) e_ = b.marg_cdf.upload(he.marg_cdf);
            if (e_ != cudaSuccess) { return fail(PBRT_E_CUDA, std::string("upload environment map: ") + cudaGetErrorString(e_)); }
            sc->upload_bytes += he.texels.size() * 16 + (he.cond_func.size() + he.cond_cdf.size() + he.cond_int.size() + he.marg_func.size() + he.marg_cdf.size()) * 4;
            DEnv de;
            std::memset(&de, 0, sizeof de);
            de.texels = b.texels.p; de.w = he.w; de.h = he.h; de.nu = he.nu; de.nv = he.nv;
            de.cond_func = b.cond_func.p; de.cond_cdf = b.cond_cdf.p; de.cond_int = b.cond_int.p;
            de.marg_func = b.marg_func.p; de.marg_cdf = b.marg_cdf.p; de.marg_int = he.marg_int;
            std::memcpy(de.l2w, l.l2w, sizeof de.l2w);
            std::memcpy(de.w2l, l.w2l, sizeof de.w2l);
            lights[inf_idx[k]].env = (uint32_t)envs.size();
            envs.push_back(de);
            sc->h_env_power[inf_idx[k]] = he.power_L;
        }
        sc->h_lights = lights;
        if (!envs.empty()) UP(envs, envs);
    }
    if (!dinst.empty()) UP(instances, dinst);
    if (any_alpha) {
        std::vector<uint2> ma(desc->n_meshes);
        for (uint32_t i = 0; i < desc->n_meshes; ++i) ma[i] = make_uint2(desc->meshes[i].alpha, desc->meshes[i].shadow_alpha);
        UP(mesh_alpha, ma);
    }
    if (desc->n_textures) {  // ImageTexture::new -> MipMap::new on the host, the pyramid levels back to back on the device
        std::vector<DTexture> dtex(desc->n_textures);
        for (uint32_t i = 0; i < desc->n_textures; ++i) {
            const PbrtTexture& t = desc->textures[i];
            if (t.kind != PBRT_TEX_IMAGE) {  // constant / scale / mix: no pyramid
                DTexture& dn = dtex[i];
                std::memset(&dn, 0, sizeof dn);
                dn.kind = t.kind;
                dn.value[0] = t.value[0]; dn.value[1] = t.channels == 1 ? t.value[0] : t.value[1]; dn.value[2] = t.channels == 1 ? t.value[0] : t.value[2];
                for (int c = 0; c < 3; ++c) dn.child[c] = t.child[c];
                sc->tex_bufs.emplace_back(new DevBuf<float4>());
                continue;
            }
            std::vector<MipLevel> pyr;
            std::vector<float> rgb3;
            const float* tex_rgb = t.texels;
            if (t.channels == 1) {  // MipMap<Float>: the same arithmetic per value, carried in three equal channels
                rgb3.resize(3 * (size_t)t.res[0] * t.res[1]);
                for (size_t q = 0; q < (size_t)t.res[0] * t.res[1]; ++q) rgb3[3 * q] = rgb3[3 * q + 1] = rgb3[3 * q + 2] = t.texels[q];
                tex_rgb = rgb3.data();
            }
            build_pyramid(tex_rgb, (int)t.res[0], (int)t.res[1], t.wrap, pyr);
            if (pyr.size() > PB_MAX_MIP_LEVELS) { return fail(PBRT_E_UNSUPPORTED, "texture pyramid deeper than 16 levels"); }
            DTexture& dt = dtex[i];
            std::memset(&dt, 0, sizeof dt);
            std::vector<float4> flat;
            for (size_t l = 0; l < pyr.size(); ++l) {
                dt.off[l] = (uint32_t)flat.size();
                for (const Sp& v : pyr[l].t) flat.push_back(make_float4(v.r, v.g, v.b, 0.0f));
            }
            sc->tex_bufs.emplace_back(new DevBuf<float4>());
            cudaError_t e_ = sc->tex_bufs.back()->upload(flat);
            if (e_ != cudaSuccess) { return fail(PBRT_E_CUDA, std::string("upload texture: ") + cudaGetErrorString(e_)); }
            sc->upload_bytes += flat.size() * 16;
            dt.texels = sc->tex_bufs.back()->p;
            dt.w = pyr[0].us; dt.h = pyr[0].vs; dt.n_levels = (int)pyr.size();
            dt.wrap = t.wrap; dt.trilinear = t.trilinear ? 1u : 0u; dt.max_anisotropy = t.max_anisotropy;
            dt.su = t.su; dt.sv = t.sv; dt.du = t.du; dt.dv = t.dv;
            dt.mapping = t.mapping;
            std::memcpy(dt.map_m, t.map_m, sizeof dt.map_m);
        }
        std::vector<float> lut(128);
        for (int i = 0; i < 128; ++i) {  // mipmap.rs:188-195
            const float alpha = 2.0f, r2 = (float)i / (float)(128 - 1);
            lut[i] = expf(-alpha * r2) - expf(-alpha);
        }
        UP(textures, dtex); UP(mat_src, mat_src); UP(ewa_lut, lut);
    }
    for (uint32_t i = 0; i < desc->n_materials; ++i) mats_single[i].cls = mats[i].cls;
    UP(materials_single, mats_single);
    UP(materials, mats); UP(lights, lights); UP(m32, m32); UP(nib, nib); UP(vdc, vdc); UP(vdci, vdci); UP(halton, halton);
#undef UP
    DScene& d = sc->d;
    std::memset(&d, 0, sizeof d);
    d.nodes = sc->nodes.p; d.n_nodes = desc->n_nodes;
    d.wide = sc->wide.p;
    d.tri_verts = sc->tri_verts.p; d.n_tris = desc->n_tris;
    d.tri_idx = sc->tri_idx.p;
    d.vn = sc->vn.p; d.vuv = sc->vuv.p; d.vs = sc->vs.p;
    d.materials = sc->materials.p; d.n_materials = desc->n_materials;
    d.lights = sc->lights.p; d.n_lights = desc->n_lights;
    d.envs = sc->envs.p; d.n_inf = n_inf;
    d.instances = sc->instances.p; d.n_instances = desc->n_instances;
    d.mesh_alpha = sc->mesh_alpha.p;
    d.textures = sc->textures.p; d.mat_src = sc->mat_src.p; d.ewa_lut = sc->ewa_lut.p; d.n_textures = desc->n_textures;
    {  // dx_camera / dy_camera, PerspectiveCamera::new (perspective.rs:82-99)
        auto r2c = [&](float x, float y) {
            const float* m = desc->camera.raster_to_camera;
            V3 r = mk3(m[0] * x + m[1] * y + m[2] * 0.0f + m[3], m[4] * x + m[5] * y + m[6] * 0.0f + m[7], m[8] * x + m[9] * y + m[10] * 0.0f + m[11]);
            const float w = m[12] * x + m[13] * y + m[14] * 0.0f + m[15];
            if (w != 1.0f) { const float inv = 1.0f / w; r = mk3(inv * r.x, inv * r.y, inv * r.z); }
            return r;
        };
        const V3 r0 = r2c(0.0f, 0.0f), dx = r2c(1.0f, 0.0f) - r0, dy = r2c(0.0f, 1.0f) - r0;
        d.dx_camera[0] = dx.x; d.dx_camera[1] = dx.y; d.dx_camera[2] = dx.z;
        d.dy_camera[0] = dy.x; d.dy_camera[1] = dy.y; d.dy_camera[2] = dy.z;
    }
    for (uint32_t k = 0; k < n_inf; ++k) d.inf[k] = inf_idx[k];
    std::memcpy(d.raster_to_camera, desc->camera.raster_to_camera, 64);
    std::memcpy(d.camera_to_world, desc->camera.camera_to_world, 64);
    d.lens_radius = desc->camera.lens_radius; d.focal_distance = desc->camera.focal_distance;
    d.shutter_open = desc->camera.shutter_open; d.shutter_close = desc->camera.shutter_close;
    for (int k = 0; k < 3; ++k) { d.wb_min[k] = desc->world_bound[k]; d.wb_max[k] = desc->world_bound[3 + k]; }
    {  // Bounds3f::bounding_sphere (geometry.rs:2079-2091)
        V3 pmin = mk3(d.wb_min[0], d.wb_min[1], d.wb_min[2]), pmax = mk3(d.wb_max[0], d.wb_max[1], d.wb_max[2]);
        V3 c = vdiv(pmin + pmax, 2.0f);
        bool inside = c.x >= pmin.x && c.x <= pmax.x && c.y >= pmin.y && c.y <= pmax.y && c.z >= pmin.z && c.z <= pmax.z;
        d.world_radius = inside ? len3(c - pmax) : 0.0f;
    }
    CK(cudaDeviceSynchronize());
    stage_lock.unlock();
    *out = sc_guard.release();
    since("done");
    return PBRT_OK;
}

static bool finite_keyframes(const PbrtAnimatedTransform& a) {
    bool ok = std::isfinite(a.start_time) && std::isfinite(a.end_time);
    for (int k = 0; k < 16; ++k)
        ok = ok && std::isfinite(a.start[k]) && std::isfinite(a.start_inv[k]) && std::isfinite(a.end[k]) && std::isfinite(a.end_inv[k]);
    return ok;
}

// m_inv is the inverse of m up to f32 rounding: every element of m * m_inv (in f64) lies within 1e-4 of the sum of the magnitudes of
// its terms of the identity's element.  A caller that hands over another matrix's inverse (or a transposed one) is caught here.
static bool inverse_pair(const float* m, const float* m_inv) {
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) {
            double p = 0.0, mag = 0.0;
            for (int k = 0; k < 4; ++k) { p += (double)m[4 * i + k] * m_inv[4 * k + j]; mag += std::fabs((double)m[4 * i + k] * m_inv[4 * k + j]); }
            if (!(std::fabs(p - (i == j ? 1.0 : 0.0)) <= 1e-4 * mag + 1e-6)) return false;
        }
    return true;
}

int pbrt_gpu_scene_create_motion(const PbrtSceneDesc* desc, const PbrtMotionDesc* motion, int device, PbrtScene** out) {
    if (!motion) return pbrt_gpu_scene_create(desc, device, out);
    if (!desc || !out) return fail(PBRT_E_INVALID, "null argument");
    *out = nullptr;
    if (motion->instances) {
        if (desc->n_instances && !desc->instances) return fail(PBRT_E_INVALID, "null instance array in scene description");
        for (uint32_t i = 0; i < desc->n_instances; ++i) {
            const PbrtAnimatedTransform& a = motion->instances[i];
            if (!finite_keyframes(a)) return fail(PBRT_E_UNSUPPORTED, "instance keyframe matrix or time is not finite");
            if (std::memcmp(a.start, desc->instances[i].m, 64) != 0 || std::memcmp(a.start_inv, desc->instances[i].m_inv, 64) != 0)
                return fail(PBRT_E_INVALID, "an instance's start keyframe differs from PbrtInstance.m / m_inv");
            for (int k = 0; k < 16; ++k)
                if (a.start[k] != a.end[k] || a.start_inv[k] != a.end_inv[k])
                    return fail(PBRT_E_UNSUPPORTED, "animated object instances are outside the GPU path");
        }
    }
    DMotion cam_mo;
    std::memset(&cam_mo, 0, sizeof cam_mo);
    if (const PbrtAnimatedTransform* c = motion->camera) {
        if (!finite_keyframes(*c)) return fail(PBRT_E_UNSUPPORTED, "camera keyframe matrix or time is not finite");
        if (std::memcmp(c->start, desc->camera.camera_to_world, 64) != 0)
            return fail(PBRT_E_INVALID, "the camera's start keyframe differs from PbrtCamera.camera_to_world");
        if (!inverse_pair(c->start, c->start_inv) || !inverse_pair(c->end, c->end_inv))
            return fail(PBRT_E_INVALID, "a camera keyframe's m_inv is not the inverse of its m");
        motion_create(c->start, c->start_inv, c->start_time, c->end, c->end_inv, c->end_time, cam_mo);
    }
    const int rc = pbrt_gpu_scene_create(desc, device, out);
    if (rc != PBRT_OK) return rc;
    // a camera whose keyframes are equal takes the static kernels: interpolate() would hand back the start transform at every time
    (*out)->cam_motion = cam_mo.actually_animated != 0;
    (*out)->cam_mo = cam_mo;
    return PBRT_OK;
}

int pbrt_gpu_host_register(const void* ptr, uint64_t bytes) {
    if (!ptr || !bytes) return fail(PBRT_E_INVALID, "null argument");
    cudaError_t e = cudaHostRegister(const_cast<void*>(ptr), (size_t)bytes, cudaHostRegisterPortable);
    if (e != cudaSuccess) { cudaGetLastError(); return fail(PBRT_E_CUDA, std::string("cudaHostRegister: ") + cudaGetErrorString(e)); }
    return PBRT_OK;
}
int pbrt_gpu_host_unregister(const void* ptr) {
    if (!ptr) return fail(PBRT_E_INVALID, "null argument");
    cudaError_t e = cudaHostUnregister(const_cast<void*>(ptr));
    if (e != cudaSuccess) { cudaGetLastError(); return fail(PBRT_E_CUDA, std::string("cudaHostUnregister: ") + cudaGetErrorString(e)); }
    return PBRT_OK;
}

uint64_t pbrt_gpu_scene_bytes(const PbrtScene* scene) { return scene ? (uint64_t)scene->upload_bytes : 0; }

void pbrt_gpu_scene_destroy(PbrtScene* scene) {
    if (!scene) return;
    cudaSetDevice(scene->device);
    delete scene;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------
// What one render call covers: a pixel rectangle, or (n_parts > 0) part `part` of the frame's 16x16 tiles dealt round robin in the
// Morton order of BlockQueue::new (blockqueue/mod.rs:33-36) -- the order the reference's worker threads take tiles in.
struct Share {
    const int32_t* rect = nullptr;
    uint32_t part = 0, n_parts = 0;
};
// Loops whose length only the device knows (the DirectLighting / Whitted recursion, path renders through null surfaces): how many
// iterations late the host reads the "work left" word.  0 = after every iteration (a stream sync per iteration); 1 = the next iteration is
// queued before the count of the current one is read, and an iteration queued past the end returns at once.  On the directlighting and
// whitted Cornell frames the three empty launches and two memsets of the extra iteration cost more than the sync they hide, so 0 is the default.
static uint32_t poll_lag() {
    if (const char* e = std::getenv("PB_POLL_LAG")) return (uint32_t)std::min(1, std::max(0, atoi(e)));
    return 0u;
}
static size_t tile_run() {
    if (const char* e = std::getenv("PB_TILE_RUN")) return (size_t)std::max(1, atoi(e));
    return 1;
}
static uint32_t morton2(uint32_t x, uint32_t y) {  // blockqueue/mod.rs morton2: interleave the low 16 bits of x and y
    auto spread = [](uint32_t v) {
        v &= 0xffffu;
        v = (v | (v << 8)) & 0x00ff00ffu;
        v = (v | (v << 4)) & 0x0f0f0f0fu;
        v = (v | (v << 2)) & 0x33333333u;
        v = (v | (v << 1)) & 0x55555555u;
        return v;
    };
    return spread(x) | (spread(y) << 1);
}
static int render_impl(PbrtScene* sc, const PbrtRenderParams* p, const Share& share, float* d_film, float* d_samples, cudaStream_t st,
                       PbrtStats* stats) {
    const bool tiled = share.n_parts > 0;
    const int32_t* rect_in = tiled ? (p ? p->sample_bounds : nullptr) : share.rect;
    if (!sc || !p || !rect_in) return fail(PBRT_E_INVALID, "null argument");
    if (tiled && share.part >= share.n_parts) return fail(PBRT_E_INVALID, "tile share out of range");
    if (tiled && d_samples) return fail(PBRT_E_INVALID, "per-sample output needs a pixel rectangle");
    // PB_TIMING=1: host wall-clock of the phases of one render call on stderr (what a frame costs besides its kernels)
    static const bool timing = getenv("PB_TIMING") && atoi(getenv("PB_TIMING"));
    const auto t_enter = std::chrono::steady_clock::now();
    auto since = [&](const char* what) {
        if (timing) fprintf(stderr, "[pb timing] dev %d %-28s %8.3f ms\n", sc->device, what, std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_enter).count());
    };
    CK(cudaSetDevice(sc->device));
    if (p->sampler > PBRT_SAMPLER_HALTON) return fail(PBRT_E_UNSUPPORTED, "sampler outside the GPU path");
    const bool halton = p->sampler == PBRT_SAMPLER_HALTON;
    if (p->spp == 0) return fail(PBRT_E_INVALID, "spp must be positive");
    if (!halton && (p->spp & (p->spp - 1)) != 0) return fail(PBRT_E_INVALID, "spp must be a power of two (SobolSampler rounds up, sobol.rs:39-45)");
    if (!(p->filter_radius[0] > 0.0f) || !(p->filter_radius[1] > 0.0f)) return fail(PBRT_E_INVALID, "filter radius must be positive");
    if (p->light_strategy > 2) return fail(PBRT_E_INVALID, "unknown light strategy");
    DRender rp;
    std::memset(&rp, 0, sizeof rp);
    for (int i = 0; i < 4; ++i) { rp.sb[i] = p->sample_bounds[i]; rp.cb[i] = p->cropped_pixel_bounds[i]; rp.pb[i] = p->pixel_bounds[i]; rp.rect[i] = rect_in[i]; }
    if (rp.rect[0] < rp.sb[0] || rp.rect[1] < rp.sb[1] || rp.rect[2] > rp.sb[2] || rp.rect[3] > rp.sb[3]) return fail(PBRT_E_INVALID, "pixel_rect outside sample_bounds");
    rp.filter_radius[0] = p->filter_radius[0]; rp.filter_radius[1] = p->filter_radius[1];
    rp.max_sample_luminance = p->max_sample_luminance;
    rp.spp = p->spp; rp.max_depth = p->max_depth; rp.rr_threshold = p->rr_threshold;
    int ext = std::max(rp.sb[2] - rp.sb[0], rp.sb[3] - rp.sb[1]);
    if (ext <= 0) return fail(PBRT_E_INVALID, "empty sample bounds");
    rp.resolution = (uint32_t)round_up_pow2_32(ext);  // sobol.rs:46-48
    rp.log2_res = 0;
    while ((1u << rp.log2_res) < rp.resolution) rp.log2_res++;
    if (rp.log2_res > 25) return fail(PBRT_E_UNSUPPORTED, "sample bounds too large for the Sobol' tables");
    const int rw = rp.rect[2] - rp.rect[0], rh = rp.rect[3] - rp.rect[1];
    std::vector<uint32_t> h_tiles;
    if (tiled && rw > 0 && rh > 0) {
        const uint32_t ntx = ((uint32_t)rw + 15u) / 16u, nty = ((uint32_t)rh + 15u) / 16u;
        if (ntx > 0xffffu || nty > 0xffffu) return fail(PBRT_E_UNSUPPORTED, "frame larger than 65535 tiles on a side");
        std::vector<std::pair<uint32_t, uint32_t>> order((size_t)ntx * nty);
        for (uint32_t ty = 0; ty < nty; ++ty)
            for (uint32_t tx = 0; tx < ntx; ++tx) order[(size_t)ty * ntx + tx] = {morton2(tx, ty), tx | (ty << 16)};
        std::sort(order.begin(), order.end());
        const size_t run = tile_run();  // consecutive Morton tiles dealt to a part at a time
        for (size_t i = 0; i < order.size(); ++i)
            if ((i / run) % share.n_parts == share.part) h_tiles.push_back(order[i].second);
    }
    const uint64_t share_pixels = tiled ? (uint64_t)h_tiles.size() * 256u : (uint64_t)std::max(rw, 0) * (uint64_t)std::max(rh, 0);
    if (share_pixels >= (1ull << 32)) return fail(PBRT_E_UNSUPPORTED, "more than 2^32 pixels in one render call");
    const uint32_t nl = sc->d.n_lights;
    // effective light strategy (lightdistrib.rs:393-418)
    uint32_t strategy = p->light_strategy;
    if (strategy == PBRT_LIGHTS_UNIFORM || nl == 1) strategy = PBRT_LIGHTS_UNIFORM;
    rp.light_strategy = strategy;

    DeviceScratch* scr = scratch_for(sc->device);
    if (!scr) return fail(PBRT_E_INVALID, "device ordinal out of range");
    std::lock_guard<std::mutex> scratch_lock(scr->mu);
    if (tiled && !h_tiles.empty()) {
        CK(scr->tiles.alloc(h_tiles.size()));
        CK(cudaMemcpyAsync(scr->tiles.p, h_tiles.data(), h_tiles.size() * 4, cudaMemcpyHostToDevice, st));  // (h_tiles outlives the render: synchronised below)
        rp.tiles = scr->tiles.p;
        rp.n_tiles = (uint32_t)h_tiles.size();
    }
    if (halton) {  // HaltonSampler::new (halton.rs:84-112)
        rp.halton = 1u;
        rp.h_center = p->sample_at_pixel_center ? 1u : 0u;
        const int res[2] = {rp.sb[2] - rp.sb[0], rp.sb[3] - rp.sb[1]};
        for (int i = 0; i < 2; ++i) {
            const int base = i == 0 ? 2 : 3;
            int scale = 1, e = 0;
            while (scale < std::min(res[i], 128)) { scale *= base; e += 1; }
            rp.h_scale[i] = (uint32_t)scale;
            rp.h_exp[i] = (uint32_t)e;
        }
        rp.h_stride = rp.h_scale[0] * rp.h_scale[1];
        rp.h_mult[0] = (uint32_t)halton_mult_inverse(rp.h_scale[1], rp.h_scale[0]);
        rp.h_mult[1] = (uint32_t)halton_mult_inverse(rp.h_scale[0], rp.h_scale[1]);
        if ((uint64_t)rp.spp * rp.h_stride >= (1ull << 32)) return fail(PBRT_E_UNSUPPORTED, "Halton sample indices beyond 2^32 (spp * 128 * 243) are outside the GPU path");
        const HaltonTables& T = halton_tables();
        if (!scr->h_dims.p) {
            CK(scr->h_dims.upload(T.dims));
            CK(scr->h_perm.upload(T.perms));
        }
        rp.h_dims = scr->h_dims.p;
        rp.h_perm = scr->h_perm.p;
    }
    cudaEvent_t ev0, ev1;
    scr->ev_used = 0;
    CK(scr->event(&ev0)); CK(scr->event(&ev1));
    std::vector<cudaEvent_t> tev, sev;  // per-launch event pairs for the trace / shade kernels
    CK(sc->counters.alloc(1));
    CK(cudaMemsetAsync(sc->counters.p, 0, sizeof(DCounters), st));
    CK(cudaEventRecord(ev0, st));
    uint32_t launches = 0, trace_launches = 0;

    if (p->integrator > PBRT_INTEGRATOR_WHITTED) return fail(PBRT_E_UNSUPPORTED, "integrator outside the GPU path");
    if (sc->d.n_textures || p->integrator >= PBRT_INTEGRATOR_DIRECT) {
        // k_texture and k_direct_step keep a DMaterial (and a texture-graph stack) in local memory: stack frames of ~1.5 KB, above the
        // default per-thread stack limit of 1 KB.  Raise it once per device (a no-op if the driver sizes known frames by itself).
        size_t cur = 0;
        CK(cudaDeviceGetLimit(&cur, cudaLimitStackSize));
        if (cur < 4096) CK(cudaDeviceSetLimit(cudaLimitStackSize, 4096));
    }
    const bool direct = p->integrator == PBRT_INTEGRATOR_DIRECT || p->integrator == PBRT_INTEGRATOR_WHITTED;
    if (direct && p->direct_strategy > PBRT_DIRECT_SAMPLE_ONE) return fail(PBRT_E_INVALID, "unknown direct-lighting strategy");
    if (p->instancing > PBRT_INSTANCING_FIXED) return fail(PBRT_E_INVALID, "unknown instancing mode");
    rp.instancing = p->instancing;
    // paths can walk through surfaces without counting a bounce (Material "none"; in PBRT_INSTANCING_REFERENCE every transformed
    // instance hit): the number of iterations is not bounded by max_depth, the queue is polled from the host.  The same loop serves a large
    // "maxdepth" (a legitimate setting: the paths then end by Russian roulette, path.rs:253-262): the fixed-length loop below would queue max_depth + 1
    // iterations over queues that have long been empty -- and never finish for the u32 maximum.
    const bool null_paths = sc->has_null_material || (sc->d.n_instances > 0 && p->instancing == PBRT_INSTANCING_REFERENCE) || rp.max_depth > 64u;
    const bool ao = p->integrator == PBRT_INTEGRATOR_AO;
    if (direct && share_pixels > 0) {
        // ---- DirectLightingIntegrator / WhittedIntegrator (pb_direct.cuh): raygen -> trace -> { k_direct_step -> k_direct_nee -> trace }
        // until every camera sample's tree is walked -> k_resolve, one batch at a time on the caller's stream.
        const bool whitted = p->integrator == PBRT_INTEGRATOR_WHITTED;
        const bool sample_all = !whitted && p->direct_strategy == PBRT_DIRECT_SAMPLE_ALL;
        const uint32_t nl = sc->d.n_lights;
        if (rp.max_depth > PB_DIRECT_MAX_DEPTH) return fail(PBRT_E_UNSUPPORTED, "direct / whitted maxdepth beyond 8 is outside the GPU path");
        std::vector<uint32_t> nee_light, nee_k, light_n(nl), light_q0(nl);
        uint32_t max_n = 1;
        for (uint32_t j = 0; j < nl; ++j) {
            light_n[j] = sample_all ? std::max(1u, sc->h_lights[j].n_samples) : 1u;
            light_q0[j] = (uint32_t)nee_light.size();
            max_n = std::max(max_n, light_n[j]);
            if (sample_all || whitted) for (uint32_t k = 0; k < light_n[j]; ++k) { nee_light.push_back(j); nee_k.push_back(k); }
        }
        if (!sample_all && !whitted) { nee_light.assign(1, 0u); nee_k.assign(1, 0u); }
        if (nee_light.empty()) { nee_light.assign(1, 0u); nee_k.assign(1, 0u); }  // no lights: k_direct_nee never has work
        const uint32_t n_nee = (uint32_t)nee_light.size();
        if (n_nee > 4096) return fail(PBRT_E_UNSUPPORTED, "more than 4096 light samples per vertex are outside the GPU path");
        DDirect dd;
        std::memset(&dd, 0, sizeof dd);
        dd.max_depth = rp.max_depth; dd.n_nee = n_nee; dd.whitted = whitted ? 1u : 0u; dd.sample_all = sample_all ? 1u : 0u;
        dd.n_arrays = sample_all ? 2u * nl * rp.max_depth : 0u;
        dd.array_end = 5u + 2u * dd.n_arrays;
        const uint64_t array_samples = (uint64_t)rp.spp * max_n;  // pixel sample numbers the 2D arrays reach
        uint32_t log2_arr = 0;
        while ((1ull << log2_arr) < array_samples) log2_arr++;
        if (halton) {
            if (array_samples * rp.h_stride >= (1ull << 32)) return fail(PBRT_E_UNSUPPORTED, "Halton sample indices beyond 2^32 are outside the GPU path");
        } else if (2u * rp.log2_res + log2_arr > 52u) return fail(PBRT_E_UNSUPPORTED, "Sobol' index beyond 52 bits");
        dd.n_chunks = std::max<uint32_t>(1u, (2u * rp.log2_res + log2_arr + 3u) / 4u);
        const bool count_work = (p->flags & PBRT_RENDER_COUNT_WORK) != 0;
        const uint64_t total_pixels = share_pixels;
        // light samples in flight per batch (PB_SIBLING_BATCH_LOG2: a test hook that forces many small batches)
        const size_t CAP = (size_t)1 << (getenv("PB_SIBLING_BATCH_LOG2") ? std::min(24, std::max(4, atoi(getenv("PB_SIBLING_BATCH_LOG2")))) : 21);
        const uint32_t paths_cap = (uint32_t)std::max<size_t>(1, std::min<size_t>((size_t)1 << 20, CAP / n_nee));
        const uint32_t samples_per_batch = std::min<uint32_t>(rp.spp, paths_cap);
        const uint32_t pixels_per_batch = (uint32_t)std::min<uint64_t>(std::max<uint32_t>(1u, paths_cap / samples_per_batch), total_pixels);
        const size_t cap = (size_t)samples_per_batch * pixels_per_batch, cap_nee = cap * n_nee, depth_n = std::max(1u, rp.max_depth);
        dd.cap = cap;
        CK(scr->filter_table.alloc(256));
        CK(cudaMemcpyAsync(scr->filter_table.p, p->filter_table, 256 * 4, cudaMemcpyHostToDevice, st));
        BatchCtx& X = scr->ctx[0];
        for (int i = 0; i < 4; ++i) CK(X.f4[i].alloc(cap));
        CK(X.rays.alloc(2 * (cap + 2 * cap_nee)));
        CK(X.sobol.alloc(cap)); CK(X.dim.alloc(cap)); CK(X.pfilm.alloc(cap));
        CK(X.queue[0].alloc(cap)); CK(X.counts.alloc(8 + PB_SHADE_CLASSES));
        DirectBufs& D = scr->direct;
        const bool dinst = sc->d.n_instances > 0;
        const bool dtex = sc->d.n_textures > 0;
        CK(D.u32.alloc(6 * cap + 2 * cap_nee + 2 * (size_t)n_nee + 2 * (size_t)std::max(1u, nl) + (dinst ? cap + cap_nee + depth_n * cap : 0) +
                       (dtex ? cap + depth_n * cap : 0)));
        CK(D.f4.alloc(4 * depth_n * cap + 4 * cap_nee + (dtex ? 3 * cap + 3 * depth_n * cap : 0)));
        uint32_t* u = D.u32.p;
        dd.state = u; u += cap; dd.depth = reinterpret_cast<int*>(u); u += cap; dd.arr_off = u; u += cap;
        dd.nee_depth = reinterpret_cast<int*>(u); u += cap; dd.nee_dim = u; u += cap; dd.nee_arr = u; u += cap;
        // (fresh shares the queue buffer, which this integrator does not use otherwise)
        dd.fresh = X.queue[0].p;
        dd.nee_flags = u; u += cap_nee; dd.nee_occl = u; u += cap_nee;
        uint32_t* t_light = u; u += n_nee; uint32_t* t_k = u; u += n_nee; uint32_t* t_n = u; u += std::max(1u, nl); uint32_t* t_q0 = u; u += std::max(1u, nl);
        uint32_t *d_hit_inst = nullptr, *d_mis_inst = nullptr;
        if (dinst) { d_hit_inst = u; u += cap; d_mis_inst = u; u += cap_nee; dd.node_inst = u; u += depth_n * cap; }
        if (dtex) { dd.cur_has_diff = u; u += cap; dd.node_has_diff = u; u += depth_n * cap; }
        CK(cudaMemcpyAsync(t_light, nee_light.data(), (size_t)n_nee * 4, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(t_k, nee_k.data(), (size_t)n_nee * 4, cudaMemcpyHostToDevice, st));
        if (nl) {
            CK(cudaMemcpyAsync(t_n, light_n.data(), (size_t)nl * 4, cudaMemcpyHostToDevice, st));
            CK(cudaMemcpyAsync(t_q0, light_q0.data(), (size_t)nl * 4, cudaMemcpyHostToDevice, st));
        }
        dd.nee_light = t_light; dd.nee_k = t_k; dd.light_n = t_n; dd.light_q0 = t_q0;
        float4* f = D.f4.p;
        dd.node_L = f; f += depth_n * cap; dd.node_mul = f; f += depth_n * cap; dd.node_hit = f; f += depth_n * cap; dd.node_rd = f; f += depth_n * cap;
        dd.nee_a = f; f += cap_nee; dd.nee_mf = f; f += cap_nee; dd.nee_md = f; f += cap_nee; dd.nee_mis_hit = f; f += cap_nee;
        if (dtex) { dd.cur_diff = f; f += 3 * cap; dd.node_diff = f; f += 3 * depth_n * cap; }
        CK(cudaStreamSynchronize(st));  // the tables above come from host vectors that go out of scope with this block's iterations
        DPaths ps;
        std::memset(&ps, 0, sizeof ps);
        ps.ray_d = dense_view(X.f4[0].p); ps.hit = dense_view(X.f4[1].p); ps.beta = dense_view(X.f4[2].p); ps.L = dense_view(X.f4[3].p);
        ps.sobol = dense_view(X.sobol.p); ps.dim = dense_view(X.dim.p); ps.p_film = X.pfilm.p;
        ps.hit_inst = d_hit_inst; ps.mis_inst = d_mis_inst;
        if (dtex) {
            CK(X.ray_diff.alloc(3 * cap)); CK(X.slot_mat.alloc(cap)); CK(X.slot_frame.alloc(2 * cap));
            ps.ray_diff = X.ray_diff.p; ps.slot_mat = X.slot_mat.p; ps.slot_frame = X.slot_frame.p;
        }
        uint32_t* d_count = X.counts.p;
        uint32_t* d_active2 = X.counts.p + 5;  // two words: iteration i counts into word i & 1, iteration i + 1 reads it
        uint32_t* d_err = X.counts.p + 2;
        uint32_t* d_nrays = X.counts.p + 3;
        uint32_t* d_cursor = X.counts.p + 4;
        CK(cudaMemsetAsync(d_err, 0, 4, st));
        TraceIO io;
        std::memset(&io, 0, sizeof io);
        io.rays = X.rays.p; io.hit = ps.hit; io.mis_hit = dense_view(dd.nee_mis_hit); io.occl = dense_view(dd.nee_occl);
        io.hit_inst = d_hit_inst; io.mis_inst = d_mis_inst; io.instancing = rp.instancing;
        DScene dsc = sc->d;
        dsc.materials = sc->materials_single.p;  // allow_multiple_lobes = false
        const int sm_count = sm_count_of(sc->device);
        TraceLauncher tl;
        CK(tl.init(sc, count_work, sm_count));
        auto trace = [&]() -> int {
            CK(cudaMemsetAsync(d_cursor, 0, 4, st));
            cudaEvent_t a, b;
            CK(scr->event(&a)); CK(scr->event(&b));
            CK(cudaEventRecord(a, st));
            tl.launch(dsc, io, d_nrays, d_cursor, sc->counters.p, st);
            CK(cudaEventRecord(b, st));
            tev.push_back(a); tev.push_back(b);
            launches++; trace_launches++;
            return PBRT_OK;
        };
        uint32_t log2_spp = 0;
        while ((1u << log2_spp) < rp.spp) log2_spp++;
        const uint32_t raygen_chunks = std::max<uint32_t>(1u, (std::min<uint32_t>(52u, 2u * rp.log2_res + log2_spp) + 3u) / 4u);
        uint32_t* h_poll = nullptr;
        cudaEvent_t poll_ev[2];
        CK(scr->poll_words(&h_poll));
        CK(scr->event(&poll_ev[0])); CK(scr->event(&poll_ev[1]));
        for (uint32_t s0 = 0; s0 < rp.spp; s0 += samples_per_batch)
            for (uint64_t pix0 = 0; pix0 < total_pixels; pix0 += pixels_per_batch) {
                BatchInfo bi;
                bi.first_pixel = (uint32_t)pix0;
                bi.n_pixels = (uint32_t)std::min<uint64_t>(pixels_per_batch, total_pixels - pix0);
                bi.first_sample = s0;
                bi.n_samples = std::min(samples_per_batch, rp.spp - s0);
                const uint32_t n = bi.n_pixels * bi.n_samples;
                CK(cudaMemsetAsync(d_nrays, 0, 4, st));
                const auto raygen = sc->cam_motion ? k_raygen<true> : k_raygen<false>;
                raygen<<<(n + 255) / 256, 256, 0, st>>>(dsc, rp, ps, bi, sc->nib.p, std::max(raygen_chunks, dd.n_chunks), sc->vdc.p, sc->vdci.p, X.queue[0].p, d_count,
                                                        X.rays.p, d_nrays, sc->counters.p, sc->cam_mo);
                launches++;
                // the recursion's length is decided on the device (the active word = camera samples that still need an iteration).  The
                // host reads that word poll_lag() iterations late (see there: 0 by default, measured): with a lag of 1 iteration i + 1 is
                // already queued when i's count arrives, and the iteration queued past the end sees the previous count at 0 and returns.
                const uint32_t lag = poll_lag();
                for (uint32_t iter = 0;; ++iter) {
                    int rc = trace();
                    if (rc != PBRT_OK) return rc;
                    uint32_t* d_active = d_active2 + (iter & 1u);
                    const uint32_t* d_prev = iter ? d_active2 + ((iter - 1u) & 1u) : nullptr;
                    CK(cudaMemsetAsync(d_nrays, 0, 4, st));
                    CK(cudaMemsetAsync(d_active, 0, 4, st));
                    cudaEvent_t e, g;
                    CK(scr->event(&e)); CK(scr->event(&g));
                    CK(cudaEventRecord(e, st));
                    k_direct_step<<<(n + 127) / 128, 128, 0, st>>>(dsc, rp, ps, dd, bi, sc->nib.p, iter == 0 ? 1u : 0u, X.rays.p, d_nrays, d_active, d_err, d_prev);
                    const uint64_t total = (uint64_t)n * n_nee;
                    k_direct_nee<<<(unsigned)((total + 127) / 128), 128, 0, st>>>(dsc, rp, ps, dd, bi, sc->nib.p, sc->vdc.p, sc->vdci.p, X.rays.p, d_nrays,
                                                                               sc->counters.p, d_err, d_prev);
                    CK(cudaEventRecord(g, st));
                    sev.push_back(e); sev.push_back(g);
                    launches += 2;
                    CK(cudaMemcpyAsync(&h_poll[iter & 1u], d_active, 4, cudaMemcpyDeviceToHost, st));
                    CK(cudaEventRecord(poll_ev[iter & 1u], st));
                    if (iter >= lag) {
                        CK(cudaEventSynchronize(poll_ev[(iter - lag) & 1u]));
                        if (h_poll[(iter - lag) & 1u] == 0u) break;
                    }
                    if (iter > 100000u) return fail(PBRT_E_CUDA, "direct integrator did not terminate");
                }
                k_resolve<<<(bi.n_pixels + 255) / 256, 256, 0, st>>>(rp, ps, bi, scr->filter_table.p, d_film, d_samples);
                launches++;
            }
        CK(cudaGetLastError());
        uint32_t h_err = 0;
        CK(cudaMemcpyAsync(&h_err, d_err, 4, cudaMemcpyDeviceToHost, st));
        CK(cudaEventRecord(ev1, st));
        CK(cudaStreamSynchronize(st));
        if (h_err) return fail(PBRT_E_UNSUPPORTED, halton ? "HaltonSampler can only sample 1000 dimensions (halton.rs:256-262)"
                                                          : "SobolSampler can only sample up to 1024 dimensions (sobol.rs:119-124)");
    } else if (ao && share_pixels > 0) {
        // ---- AOIntegrator (integrators/ao.rs): raygen -> trace -> k_ao_shade (ao_n any-hit rays per camera sample) -> trace ->
        // k_ao_resolve -> k_resolve, one batch at a time on the caller's stream.
        const uint32_t ao_n = p->ao_samples;
        if (ao_n == 0 || ao_n > 4096) return fail(PBRT_E_INVALID, "ao nsamples out of range (1..4096)");
        const uint64_t array_samples = (uint64_t)rp.spp * ao_n;  // pixel sample numbers the 2D array reaches
        uint32_t log2_arr = 0;
        while ((1ull << log2_arr) < array_samples) log2_arr++;
        if (halton) {
            if (array_samples * rp.h_stride >= (1ull << 32)) return fail(PBRT_E_UNSUPPORTED, "Halton sample indices beyond 2^32 are outside the GPU path");
        } else if (2u * rp.log2_res + log2_arr > 52u) return fail(PBRT_E_UNSUPPORTED, "Sobol' index beyond 52 bits");
        const uint32_t n_chunks = std::max<uint32_t>(1u, (2u * rp.log2_res + log2_arr + 3u) / 4u);
        const bool count_work = (p->flags & PBRT_RENDER_COUNT_WORK) != 0;
        const uint64_t total_pixels = share_pixels;
        const size_t CAP = (size_t)1 << (getenv("PB_SIBLING_BATCH_LOG2") ? std::min(24, std::max(4, atoi(getenv("PB_SIBLING_BATCH_LOG2")))) : 22);  // any-hit rays in flight per batch
        const uint32_t paths_cap = (uint32_t)std::max<size_t>(1, CAP / ao_n);
        const uint32_t samples_per_batch = std::min<uint32_t>(rp.spp, paths_cap);
        const uint32_t pixels_per_batch = (uint32_t)std::min<uint64_t>(std::max<uint32_t>(1u, paths_cap / samples_per_batch), total_pixels);
        const size_t cap_paths = (size_t)samples_per_batch * pixels_per_batch, cap_rays = cap_paths * ao_n;
        CK(scr->filter_table.alloc(256));
        CK(cudaMemcpyAsync(scr->filter_table.p, p->filter_table, 256 * 4, cudaMemcpyHostToDevice, st));
        BatchCtx& X = scr->ctx[0];
        for (int i = 0; i < 4; ++i) CK(X.f4[i].alloc(cap_paths));
        CK(X.rays.alloc(2 * std::max(cap_paths, cap_rays)));
        CK(X.occl.alloc(cap_rays)); CK(X.ao_weight.alloc(cap_rays));
        CK(X.sobol.alloc(cap_paths)); CK(X.dim.alloc(cap_paths)); CK(X.pfilm.alloc(cap_paths));
        CK(X.queue[0].alloc(cap_paths)); CK(X.counts.alloc(8 + PB_SHADE_CLASSES));
        DPaths ps;
        std::memset(&ps, 0, sizeof ps);
        ps.ray_d = dense_view(X.f4[0].p); ps.hit = dense_view(X.f4[1].p); ps.beta = dense_view(X.f4[2].p); ps.L = dense_view(X.f4[3].p);
        ps.occl = dense_view(X.occl.p); ps.sobol = dense_view(X.sobol.p); ps.dim = dense_view(X.dim.p); ps.p_film = X.pfilm.p;
        const bool ainst = sc->d.n_instances > 0;  // two-level traversal; the any-hit rays need no instance record of their own
        if (ainst) { CK(X.hit_inst.alloc(std::max(cap_paths, cap_rays))); ps.hit_inst = X.hit_inst.p; }
        uint32_t* d_count = X.counts.p;
        uint32_t* d_nrays = X.counts.p + 3;
        uint32_t* d_cursor = X.counts.p + 4;
        TraceIO io;
        std::memset(&io, 0, sizeof io);
        io.rays = X.rays.p; io.hit = ps.hit; io.mis_hit = ps.hit; io.occl = ps.occl;
        io.hit_inst = ps.hit_inst; io.mis_inst = ps.hit_inst; io.instancing = rp.instancing;
        const int sm_count = sm_count_of(sc->device);
        TraceLauncher tl;
        CK(tl.init(sc, count_work, sm_count));
        auto trace = [&]() -> int {
            CK(cudaMemsetAsync(d_cursor, 0, 4, st));
            cudaEvent_t a, b;
            CK(scr->event(&a)); CK(scr->event(&b));
            CK(cudaEventRecord(a, st));
            tl.launch(sc->d, io, d_nrays, d_cursor, sc->counters.p, st);
            CK(cudaEventRecord(b, st));
            tev.push_back(a); tev.push_back(b);
            launches++; trace_launches++;
            return PBRT_OK;
        };
        for (uint32_t s0 = 0; s0 < rp.spp; s0 += samples_per_batch)
            for (uint64_t pix0 = 0; pix0 < total_pixels; pix0 += pixels_per_batch) {
                BatchInfo bi;
                bi.first_pixel = (uint32_t)pix0;
                bi.n_pixels = (uint32_t)std::min<uint64_t>(pixels_per_batch, total_pixels - pix0);
                bi.first_sample = s0;
                bi.n_samples = std::min(samples_per_batch, rp.spp - s0);
                const uint32_t n = bi.n_pixels * bi.n_samples;
                CK(cudaMemsetAsync(d_nrays, 0, 4, st));
                const auto raygen = sc->cam_motion ? k_raygen<true> : k_raygen<false>;
                raygen<<<(n + 255) / 256, 256, 0, st>>>(sc->d, rp, ps, bi, sc->nib.p, n_chunks, sc->vdc.p, sc->vdci.p, X.queue[0].p, d_count, X.rays.p, d_nrays,
                                                        sc->counters.p, sc->cam_mo);
                launches++;
                int rc = trace();
                if (rc != PBRT_OK) return rc;
                CK(cudaMemsetAsync(d_nrays, 0, 4, st));
                cudaEvent_t e, f;
                CK(scr->event(&e)); CK(scr->event(&f));
                CK(cudaEventRecord(e, st));
                const uint64_t total = (uint64_t)n * ao_n;
                k_ao_shade<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(sc->d, rp, ps, bi, ao_n, p->ao_cos_sample ? 1u : 0u, sc->nib.p, n_chunks, sc->vdc.p,
                                                                         sc->vdci.p, X.rays.p, X.ao_weight.p, d_nrays);
                CK(cudaEventRecord(f, st));
                sev.push_back(e); sev.push_back(f);
                launches++;
                if ((rc = trace()) != PBRT_OK) return rc;
                k_ao_resolve<<<(n + 255) / 256, 256, 0, st>>>(ps, bi, ao_n, X.ao_weight.p, X.occl.p);
                k_resolve<<<(bi.n_pixels + 255) / 256, 256, 0, st>>>(rp, ps, bi, scr->filter_table.p, d_film, d_samples);
                launches += 2;
            }
        CK(cudaGetLastError());
        CK(cudaEventRecord(ev1, st));
        CK(cudaStreamSynchronize(st));
    } else if (share_pixels > 0) {
        const uint64_t total_pixels = share_pixels;
        // Camera samples in flight per batch.  2^24 (6 GB of wavefront state per stream context): every batch ends in one or two iterations
        // that hold a few thousand rays and still last as long as one ray's chain of dependent fetches, so fewer, larger batches spend
        // less of the frame in those tails (the statue and shares of its frame gain; Cornell and the conference scene are indifferent).
        // Two contexts of 2^24 take 12 GB, well inside an 80 GB H100.
        // Scenes with textured materials stay at 2^22: k_texture leaves a 496-byte lobe record per hit (8 GB per context at 2^24) that k_shade
        // reads back through the class-sorted queue, and k_shade's time per slot grows with that working set.
        static const int cap_log2_env = getenv("PB_BATCH_LOG2") ? std::min(26, std::max(10, atoi(getenv("PB_BATCH_LOG2")))) : 0;
        const int cap_log2 = cap_log2_env ? cap_log2_env : (sc->d.n_textures ? 22 : 24);
        const size_t CAP = (size_t)1 << cap_log2;
        const uint32_t samples_per_batch = (uint32_t)std::min<size_t>(rp.spp, CAP);
        const uint32_t pixels_per_batch = (uint32_t)std::min<uint64_t>(std::max<size_t>(1, CAP / samples_per_batch), total_pixels);
        const size_t cap = (size_t)samples_per_batch * pixels_per_batch;
        const uint64_t n_batches = ((rp.spp + samples_per_batch - 1) / samples_per_batch) * ((total_pixels + pixels_per_batch - 1) / pixels_per_batch);
        // PB_SHADE_SPEC=0 turns the single-lobe instantiations of k_shade off (A/B switch; every class then runs the general one);
        // =1 keeps only the Lambert one (round 2's first step)
        static const int shade_spec = getenv("PB_SHADE_SPEC") ? atoi(getenv("PB_SHADE_SPEC")) : 2;
        const bool plan_instanced = sc->d.n_instances > 0;
        struct ShadeLaunch { int spec; uint32_t lo, hi; };
        std::vector<ShadeLaunch> shade_plan;
        {
            uint32_t mask = sc->class_mask & ~1u, covered = 0;
            const uint32_t first_general = PB_SPEC_PLASTIC + 1;
            for (uint32_t c = 1; c < first_general && shade_spec; ++c) {
                if (!(mask & (1u << c))) continue;
                const bool have = c == 1 + LOBE_LAMBERT || (shade_spec >= 2 && !halton && !plan_instanced && (c == 1 + LOBE_SPEC_REFL || c == 1 + LOBE_FRESNEL_SPEC || c == 1 + LOBE_OREN_NAYAR ||
                                                                                                    c == 1 + LOBE_MF_REFL || c == 1 + LOBE_FRESNEL_BLEND || c == PB_SPEC_PLASTIC));
                if (!have) continue;
                shade_plan.push_back({(int)c, c, c + 1});
                covered |= 1u << c;
            }
            // the classes no specialised launch covers, as maximal runs, for the general instantiation
            const uint32_t rest = mask & ~covered;
            for (uint32_t c = 1; c < PB_SHADE_CLASSES;) {
                if (!(rest & (1u << c))) { ++c; continue; }
                uint32_t e = c;
                while (e < PB_SHADE_CLASSES && (rest & (1u << e))) ++e;
                shade_plan.push_back({0, c, e});
                c = e;
            }
            // when no material has class 1, the null-material hits that k_sort files under class 1 (a shape without a material, or a
            // moved instance under quirk Q7): folded into the Lambert launch when nothing lies between, else a launch of their own (the
            // cheapest instantiation: no BSDF is touched).  An otherwise empty plan keeps that launch too: k_shade resets the counters
            // the next iteration fills.
            const uint32_t lam = 1 + LOBE_LAMBERT;
            const bool null_hits = sc->has_null_material || (plan_instanced && p->instancing == PBRT_INSTANCING_REFERENCE);
            if (!(mask & 2u) && (null_hits || shade_plan.empty())) {
                bool folded = false;
                if ((covered & (1u << lam)) && (mask & ((1u << lam) - 4u)) == 0u)
                    for (ShadeLaunch& l : shade_plan) if (l.spec == (int)lam) { l.lo = 1; folded = true; }
                if (!folded) shade_plan.insert(shade_plan.begin(), ShadeLaunch{shade_spec ? (int)lam : 0, 1u, 2u});
            }
        }
        // Two batches in flight on two streams: k_trace and k_shade leave the SMs idle in different ways, so letting one batch
        // trace while the other shades fills the SMs better than either alone.  Disabled for the roofline timing pass
        // (PBRT_RENDER_SINGLE_STREAM: kernel durations must not be inflated by a co-resident kernel), when the queue
        // has to be polled from the host (null materials), and when there is only one batch.
        static const bool dual_env = !(getenv("PB_SINGLE_STREAM") && atoi(getenv("PB_SINGLE_STREAM")));
        // ... and when an iteration is a single k_shade launch.  On an H100 at 400 W (DESIGN.md section 7) the statue, two launches per
        // iteration, renders at 1 629-1 637 Mrays/s with two batches in flight against 1 574-1 585 with one; Cornell, one Lambert launch,
        // cannot be told apart (2 873-2 953 against 2 902-2 969), so it keeps one stream.  PB_STREAMS = 1 keeps one batch in flight,
        // PB_STREAMS >= 2 forces two.
        // A textured frame is bound by k_texture's per-hit records (written once, read back by k_shade): a second batch in flight doubles that
        // working set and loses.
        const bool streams_forced = getenv("PB_STREAMS") && atoi(getenv("PB_STREAMS")) >= 2;
        const bool dual = dual_env && !(p->flags & PBRT_RENDER_SINGLE_STREAM) && !null_paths && n_batches > 1 &&
                          !(getenv("PB_STREAMS") && atoi(getenv("PB_STREAMS")) <= 1) && ((shade_plan.size() >= 2 && sc->d.n_textures == 0) || streams_forced);
        static const int streams_env = getenv("PB_STREAMS") ? std::min(4, std::max(1, atoi(getenv("PB_STREAMS")))) : 2;
        const int n_ctx = dual ? (int)std::min<uint64_t>((uint64_t)streams_env, n_batches) : 1;

        const int sm_count = sm_count_of(sc->device);
        const bool count_work = (p->flags & PBRT_RENDER_COUNT_WORK) != 0;
        const bool spatial = strategy == PBRT_LIGHTS_SPATIAL && nl > 0;

        // ---- light grid geometry (SpatialLightDistribution::new lightdistrib.rs:127-150) / fixed distributions ----
        int nv[3] = {1, 1, 1};
        size_t nvox = 1;
        if (spatial) {
            float diag[3] = {sc->d.wb_max[0] - sc->d.wb_min[0], sc->d.wb_max[1] - sc->d.wb_min[1], sc->d.wb_max[2] - sc->d.wb_min[2]};
            int me = (diag[0] > diag[1] && diag[0] > diag[2]) ? 0 : (diag[1] > diag[2] ? 1 : 2);
            float bmax = diag[me];
            for (int i = 0; i < 3; ++i) {
                nv[i] = std::max(1, f2i_sat(roundf(diag[i] / bmax * 64.0f)));
                nvox *= (size_t)nv[i];
            }
        }
        // func + contrib + cdf + func_int of one voxel.  Dense tables for every voxel are the fast path (Cornell: 7 MB); with one
        // light per emissive triangle they would be nvox x n_lights x 12 bytes (10 k emitters: 31 GB per stream context), so above
        // the budget the tables become rows handed out on first touch (DLightGrid::row) and the render fails, rather than the
        // allocation, should the paths visit more voxels than fit.
        const size_t grid_row_bytes = (3 * std::max<size_t>(nl, 1) + 2) * sizeof(float);
        const size_t grid_budget = lightgrid_budget();
        const bool grid_sparse = spatial && nvox * grid_row_bytes > grid_budget;
        const size_t grid_rows = grid_sparse ? std::max<size_t>(1, std::min(nvox, grid_budget / grid_row_bytes)) : nvox;
        std::vector<float> fixed_f(nl, 1.0f), fixed_cdf;
        float fixed_int = 0.0f;
        if (!spatial && nl > 0) {
            if (strategy == PBRT_LIGHTS_POWER)  // compute_light_power_distribution integrator.rs:574-584, diffuse.rs:85-93
                for (uint32_t j = 0; j < nl; ++j) {
                    const DLight& l = sc->h_lights[j];
                    Sp pw;
                    const Sp I = mksp(l.L[0], l.L[1], l.L[2]);
                    if (l.kind == PBRT_LIGHT_POINT) pw = I * (4.0f * PB_PI);  // point.rs / spot.rs / distant.rs power()
                    else if (l.kind == PBRT_LIGHT_SPOT) pw = I * 2.0f * PB_PI * (1.0f - 0.5f * (l.cos_falloff_start + l.cos_total_width));
                    else if (l.kind == PBRT_LIGHT_DISTANT) pw = I * PB_PI * sc->d.world_radius * sc->d.world_radius;
                    else if (l.kind == PBRT_LIGHT_INFINITE) pw = sc->h_env_power[j] * sp1(PB_PI * sc->d.world_radius * sc->d.world_radius);  // infinite.rs:349-355
                    else pw = I * (l.two_sided ? 2.0f : 1.0f) * l.area * PB_PI;
                    fixed_f[j] = lum(pw);
                }
            make_distribution(fixed_f, fixed_cdf, fixed_int);
        }
        CK(scr->filter_table.alloc(256));
        CK(cudaMemcpyAsync(scr->filter_table.p, p->filter_table, 256 * 4, cudaMemcpyHostToDevice, st));

        // Sobol' dimensions reachable by this render: 5 camera dims + 8 per shaded bounce; index bits: 2*log2(resolution)
        // pixel bits + log2(spp) sample bits (sobol_interval_to_index)
        uint32_t dims_needed = (uint32_t)std::min<uint64_t>(1024u, 5 + 8 * ((uint64_t)rp.max_depth + 1));
        uint32_t log2_spp = 0;
        while ((1u << log2_spp) < rp.spp) log2_spp++;
        const uint32_t index_bits = std::min<uint32_t>(52u, 2u * rp.log2_res + log2_spp);
        const uint32_t n_chunks = std::max<uint32_t>(1u, (index_bits + 3u) / 4u);
        // this render's transposed nibble-table slice nibT[(chunk*16+e)*ds + dim], padded by 8 dimensions (pb_sobol.cuh)
        const uint32_t sobol_ds = (dims_needed + 8u) | 1u;
        {
            std::vector<uint32_t>& T = scr->h_nibT;
            T.assign((size_t)n_chunks * 16 * sobol_ds, 0u);
            for (uint32_t c = 0; c < n_chunks; ++c)
                for (uint32_t e = 0; e < 16; ++e)
                    for (uint32_t d = 0; d < dims_needed; ++d) T[((size_t)c * 16 + e) * sobol_ds + d] = sc->h_nib[((size_t)d * PB_SOBOL_CHUNKS + c) * 16 + e];
            CK(scr->nibT.alloc(T.size()));
            CK(cudaMemcpyAsync(scr->nibT.p, T.data(), T.size() * 4, cudaMemcpyHostToDevice, st));
        }
        const bool stage_sobol = (size_t)sobol_ds * n_chunks * 64 <= PB_SMEM_SOBOL_BYTES;
        const uint32_t sobol_cfg = sobol_ds | (stage_sobol ? 0x80000000u : 0u);
        const size_t shade_smem = stage_sobol ? (size_t)sobol_ds * n_chunks * 64 : 0;
        const uint32_t* shade_nib = scr->nibT.p;
        // persistent trace grid: the CTAs that are resident at once (half of them per stream when two batches overlap)
        const bool instanced = sc->d.n_instances > 0;
        const bool textured = sc->d.n_textures > 0;
        TraceLauncher tl;
        CK(tl.init(sc, count_work, sm_count));
        tl.grid = sm_count * std::max(1, std::max(tl.blocks_per_sm, 1) / n_ctx);
        const int shade_grid = sm_count * (8 / n_ctx);
        int shade_grid_spec = shade_grid;
        if (shade_spec) {
            int bps = 4;
            cudaError_t oe;
            constexpr int L = 1 + LOBE_LAMBERT;
            if (halton) oe = instanced ? cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, k_shade<false, true, true, L>, PB_SHADE_THREADS, 0)
                            : sc->area_only ? cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, k_shade<true, true, false, L>, PB_SHADE_THREADS, 0)
                                            : cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, k_shade<false, true, false, L>, PB_SHADE_THREADS, 0);
            else oe = instanced ? cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, k_shade<false, false, true, L>, PB_SHADE_THREADS, shade_smem)
                     : sc->area_only ? cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, k_shade<true, false, false, L>, PB_SHADE_THREADS, shade_smem)
                                     : cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, k_shade<false, false, false, L>, PB_SHADE_THREADS, shade_smem);
            CK(oe);
            shade_grid_spec = sm_count * std::max(1, std::max(bps, 1) / n_ctx);
        }
        // the launches of one k_shade step: {specialisation, first class, one past the last class}.  Every single-lobe class the scene has
        // gets its own instantiation (the Lambert one exists for every sampler / light / instancing combination, the others for the Sobol'
        // sampler without instances: what the benchmark configurations run); class 0 ("nothing to shade") and the null-material hits of
        // class 1 ride with the first launch; what is left goes to the general instantiation.
        // ---- per-context buffers ---------------------------------------------------------------
        struct Live {
            DPaths ps; DLightGrid grid; TraceIO io;
            uint32_t *counts, *d_err, *d_nrays, *d_cursor, *d_cls_count;
            cudaStream_t s;
            int cur;
            int iter;
        } live[4];
        // PB_RAY_SORT=1 switches the coherence order of the ray queues on.  It shortens k_trace on Cornell and the conference scene
        // (not on the 4.3 M-triangle statue), but the three bucketing kernels cost more than that (they re-read the 32 B ray records and fight over a few hot histogram bins), so it is OFF by default until
        // the keys are produced by k_shade and the histogram is warp-aggregated (DESIGN.md section 9).
        static const int ray_sort_mode = getenv("PB_RAY_SORT") ? atoi(getenv("PB_RAY_SORT")) : 0;  // 2: two-level scatter
        static const bool ray_sort = ray_sort_mode != 0;
        // PB_STATE_AOS=0: one dense array per state field instead of the three interleaved records (A/B switch)
        static const bool state_aos = !(getenv("PB_STATE_AOS") && atoi(getenv("PB_STATE_AOS")) == 0);
        // PB_RAY_PREP=1: k_rayprep computes the per-ray traversal constants ahead of k_trace (experiment, see pb_kernels.cuh)
        static const bool ray_prep = getenv("PB_RAY_PREP") && atoi(getenv("PB_RAY_PREP"));
        static const uint32_t ray_key_mask = getenv("PB_RAY_KEY_MASK") ? (uint32_t)strtoul(getenv("PB_RAY_KEY_MASK"), nullptr, 0) : 0x1fffu;
        cudaEvent_t ev_start;
        CK(scr->event(&ev_start));
        CK(cudaEventRecord(ev_start, st));
        for (int c = 0; c < n_ctx; ++c) {
            BatchCtx& X = scr->ctx[c];
            Live& V = live[c];
            if (dual) {
                if (!X.stream) CK(cudaStreamCreateWithFlags(&X.stream, cudaStreamNonBlocking));
                V.s = X.stream;
                CK(cudaStreamWaitEvent(V.s, ev_start, 0));
            } else V.s = st;
            if (state_aos) { for (int i = 0; i < 3; ++i) CK(X.rec[i].alloc(4 * cap)); CK(X.f4[3].alloc(cap)); }
            else {
                for (int i = 0; i < 9; ++i) CK(X.f4[i].alloc(cap));
                CK(X.occl.alloc(cap)); CK(X.sobol.alloc(cap)); CK(X.dim.alloc(cap));
            }
            CK(X.rays.alloc(2 * 3 * cap));  // up to three rays (path, MIS, shadow) per slot and bounce
            CK(X.pfilm.alloc(cap));
            CK(X.queue[0].alloc(cap)); CK(X.queue[1].alloc(cap)); CK(X.counts.alloc(8 + 2 * PB_SHADE_CLASSES));
            CK(X.cls_queue.alloc((size_t)PB_SHADE_CLASSES * cap));
            CK(X.g_state.alloc(nvox)); CK(X.g_func.alloc(grid_rows * std::max<size_t>(nl, 1))); CK(X.g_cdf.alloc(grid_rows * (nl + 1)));
            CK(X.g_fint.alloc(grid_rows)); CK(X.g_contrib.alloc(grid_rows * std::max<size_t>(nl, 1))); CK(X.g_request.alloc(nvox + 3));
            if (grid_sparse) CK(X.g_row.alloc(nvox));
            DPaths& ps = V.ps;
            if (state_aos) {  // three 64-byte records per slot (pb_scene.cuh::DPaths)
                auto f4 = [](float4* base, int k) { StridedView<float4> v; v.p = base + k; v.stride = 4; return v; };
                float4 *A = X.rec[0].p, *B = X.rec[1].p, *C = X.rec[2].p;
                // (L + flags stay a dense array: k_sort reads the flags word of every slot and k_resolve walks L in slot order)
                ps.L = dense_view(X.f4[3].p); ps.ray_d = f4(A, 1); ps.beta = f4(A, 2);
                ps.sobol.p = reinterpret_cast<uint2*>(A + 3); ps.sobol.stride = 8;
                ps.dim.p = reinterpret_cast<uint32_t*>(A + 3) + 2; ps.dim.stride = 16;
                ps.ld_light = f4(B, 0); ps.mis_d = f4(B, 1); ps.mis_f = f4(B, 2); ps.nee_beta = f4(B, 3);
                ps.hit = f4(C, 0); ps.mis_hit = f4(C, 1);
                ps.occl.p = reinterpret_cast<uint32_t*>(C + 2); ps.occl.stride = 16;
            } else {
                ps.ray_d = dense_view(X.f4[0].p); ps.hit = dense_view(X.f4[1].p); ps.beta = dense_view(X.f4[2].p); ps.L = dense_view(X.f4[3].p);
                ps.ld_light = dense_view(X.f4[4].p); ps.mis_hit = dense_view(X.f4[5].p); ps.mis_d = dense_view(X.f4[6].p); ps.mis_f = dense_view(X.f4[7].p);
                ps.nee_beta = dense_view(X.f4[8].p);
                ps.occl = dense_view(X.occl.p); ps.sobol = dense_view(X.sobol.p); ps.dim = dense_view(X.dim.p);
            }
            ps.p_film = X.pfilm.p;
            if (instanced) { CK(X.hit_inst.alloc(cap)); CK(X.mis_inst.alloc(cap)); }
            ps.hit_inst = X.hit_inst.p; ps.mis_inst = X.mis_inst.p;
            ps.ray_diff = nullptr; ps.slot_mat = nullptr; ps.slot_frame = nullptr;
            if (textured) {
                CK(X.ray_diff.alloc(3 * cap)); CK(X.slot_mat.alloc(cap)); CK(X.slot_frame.alloc(2 * cap));
                ps.ray_diff = X.ray_diff.p; ps.slot_mat = X.slot_mat.p; ps.slot_frame = X.slot_frame.p;
            }
            DLightGrid& g = V.grid;
            std::memset(&g, 0, sizeof g);
            g.n_lights = (int)nl;
            g.nv[0] = nv[0]; g.nv[1] = nv[1]; g.nv[2] = nv[2];
            g.state = X.g_state.p; g.func = X.g_func.p; g.cdf = X.g_cdf.p; g.func_int = X.g_fint.p;
            g.contrib = X.g_contrib.p; g.request = X.g_request.p; g.n_request = X.g_request.p + nvox;
            g.row = grid_sparse ? X.g_row.p : nullptr;
            g.max_rows = (uint32_t)grid_rows;
            CK(cudaMemsetAsync(g.state, 0, nvox * sizeof(int), V.s));
            CK(cudaMemsetAsync(g.n_request, 0, 3 * sizeof(uint32_t), V.s));
            if (grid_sparse) CK(cudaMemsetAsync(g.row, 0, nvox * sizeof(int), V.s));
            if (!spatial && nl > 0) {
                CK(cudaMemcpyAsync(g.func, fixed_f.data(), nl * 4, cudaMemcpyHostToDevice, V.s));
                CK(cudaMemcpyAsync(g.cdf, fixed_cdf.data(), (nl + 1) * 4, cudaMemcpyHostToDevice, V.s));
                CK(cudaMemcpyAsync(g.func_int, &fixed_int, 4, cudaMemcpyHostToDevice, V.s));
            }
            V.counts = X.counts.p; V.d_err = X.counts.p + 2; V.d_nrays = X.counts.p + 3; V.d_cursor = X.counts.p + 4; V.d_cls_count = X.counts.p + 8;
            CK(cudaMemsetAsync(X.counts.p, 0, (8 + 2 * PB_SHADE_CLASSES) * sizeof(uint32_t), V.s));
            std::memset(&V.io, 0, sizeof V.io);
            V.io.rays = X.rays.p; V.io.hit = ps.hit; V.io.mis_hit = ps.mis_hit; V.io.occl = ps.occl;
            V.io.hit_inst = ps.hit_inst; V.io.mis_inst = ps.mis_inst; V.io.instancing = rp.instancing;
            V.cur = 0;
            if (ray_sort) { CK(X.ray_keys.alloc(3 * cap)); CK(X.ray_perm.alloc(3 * cap)); CK(X.ray_hist.alloc(PB_RAY_KEYS)); }
            if (ray_prep) CK(X.rays_pre.alloc(2 * 3 * cap));
        }

        // ---- one iteration (trace -> sort -> light grid -> shade) of the batch living in context c ----
        // `stagger` (first iteration of a batch pair): context 1 starts tracing only when context 0 has finished its
        // first trace, so that from then on one batch traces while the other shades
        cudaEvent_t ev_stagger[4];
        for (int i = 0; i < 4; ++i) CK(scr->event(&ev_stagger[i]));
        auto enqueue_iteration = [&](int c, bool stagger) -> int {
            BatchCtx& X = scr->ctx[c];
            Live& V = live[c];
            cudaStream_t s = V.s;
            const int cur = V.cur;
            uint32_t* c_in = V.counts + cur;
            uint32_t* c_out = V.counts + (cur ^ 1);
            uint32_t* cls_now = V.d_cls_count + PB_SHADE_CLASSES * (V.iter & 1);        // filled by this iteration's k_sort
            uint32_t* cls_next = V.d_cls_count + PB_SHADE_CLASSES * ((V.iter + 1) & 1);  // cleared by this iteration's k_shade
            if (stagger && c >= 1) CK(cudaStreamWaitEvent(s, ev_stagger[c - 1], 0));
            // camera rays arrive in pixel order (coherent as they are); every later queue is bucketed by direction / origin
            V.io.perm = nullptr;
            if (ray_sort && V.iter > 0) {
                CK(cudaMemsetAsync(X.ray_hist.p, 0, PB_RAY_KEYS * sizeof(uint32_t), s));
                k_ray_hist<<<sm_count * 4, 256, 0, s>>>(V.d_nrays, X.ray_keys.p, X.ray_hist.p);
                k_ray_scan<<<1, 1024, 0, s>>>(X.ray_hist.p);
                if (ray_sort_mode == 2) k_ray_scatter2<<<sm_count * 8, 256, 0, s>>>(V.d_nrays, X.ray_keys.p, X.ray_hist.p, X.ray_perm.p);
                else k_ray_scatter<<<sm_count * 8, 256, 0, s>>>(V.d_nrays, X.ray_keys.p, X.ray_hist.p, X.ray_perm.p);
                launches += 3;
                V.io.perm = X.ray_perm.p;
            }
            V.iter++;
            cudaEvent_t a, b;
            CK(scr->event(&a)); CK(scr->event(&b));
            CK(cudaEventRecord(a, s));
            V.io.pre = nullptr;
            if (ray_prep) {  // (inside the k_trace event pair: its cost counts as traversal time)
                k_rayprep<<<sm_count * 8, 256, 0, s>>>(X.rays.p, V.d_nrays, X.rays_pre.p);
                launches++;
                V.io.pre = X.rays_pre.p;
            }
            tl.launch(sc->d, V.io, V.d_nrays, V.d_cursor, sc->counters.p, s);
            CK(cudaEventRecord(b, s));
            if (stagger) CK(cudaEventRecord(ev_stagger[c], s));
            tev.push_back(a); tev.push_back(b);
            launches++; trace_launches++;
            k_sort<<<sm_count * 8, 256, 0, s>>>(sc->d, V.ps, V.grid, spatial ? 1u : 0u, rp.instancing, X.queue[cur].p, c_in, X.cls_queue.p, (uint32_t)cap, cls_now, c_out,
                                                V.d_nrays);
            launches++;
            if (textured) {  // V.iter == 1: the rays just traced are the camera rays, the only ones with differentials
                k_texture<<<sm_count * 8, 128, 0, s>>>(sc->d, rp, V.ps, X.queue[cur].p, c_in, V.iter == 1 ? 1u : 0u);
                launches++;
            }
            if (spatial) {
                k_lightgrid_contrib<<<sm_count * 2, 128, 0, s>>>(sc->d, V.grid, sc->halton.p);
                k_lightgrid_build<<<sm_count, 128, 0, s>>>(V.grid);
                launches += 2;
            }
            cudaEvent_t e, f;
            CK(scr->event(&e)); CK(scr->event(&f));
            CK(cudaEventRecord(e, s));
#define PB_SHADE_ARGS(lo, hi) (sc->d, rp, V.ps, V.grid, shade_nib, sobol_cfg, n_chunks, X.cls_queue.p, (uint32_t)cap, cls_now, X.queue[cur ^ 1].p, c_out, \
                              X.rays.p, V.d_nrays, sc->counters.p, V.d_err, ray_sort ? X.ray_keys.p : nullptr, ray_key_mask, V.d_cursor,    \
                              spatial ? V.grid.n_request : nullptr, cls_next, (uint32_t)(lo), (uint32_t)(hi))
#define PB_SHADE_LAUNCH(SPEC, grid, lo, hi)                                                                                                   \
    do {                                                                                                                                      \
        /* instanced scenes take the general-light variants (an instanced scene lit by area lights alone is rare enough) */                   \
        if (halton) {                                                                                                                         \
            if (instanced) k_shade<false, true, true, SPEC><<<grid, PB_SHADE_THREADS, 0, s>>>PB_SHADE_ARGS(lo, hi);                            \
            else if (sc->area_only) k_shade<true, true, false, SPEC><<<grid, PB_SHADE_THREADS, 0, s>>>PB_SHADE_ARGS(lo, hi);                   \
            else k_shade<false, true, false, SPEC><<<grid, PB_SHADE_THREADS, 0, s>>>PB_SHADE_ARGS(lo, hi);                                     \
        } else {                                                                                                                              \
            if (instanced) k_shade<false, false, true, SPEC><<<grid, PB_SHADE_THREADS, shade_smem, s>>>PB_SHADE_ARGS(lo, hi);                  \
            else if (sc->area_only) k_shade<true, false, false, SPEC><<<grid, PB_SHADE_THREADS, shade_smem, s>>>PB_SHADE_ARGS(lo, hi);         \
            else k_shade<false, false, false, SPEC><<<grid, PB_SHADE_THREADS, shade_smem, s>>>PB_SHADE_ARGS(lo, hi);                           \
        }                                                                                                                                     \
        launches++;                                                                                                                           \
    } while (0)
            for (const ShadeLaunch& sl : shade_plan) {
                switch (sl.spec) {
                    case 1 + LOBE_LAMBERT: PB_SHADE_LAUNCH(1 + LOBE_LAMBERT, shade_grid_spec, sl.lo, sl.hi); break;
#define PB_SHADE_SOBOL_ONLY(SPEC)                                                                                                                         \
    do {                                                                                                                                                  \
        if (sc->area_only) k_shade<true, false, false, SPEC><<<shade_grid, PB_SHADE_THREADS, shade_smem, s>>>PB_SHADE_ARGS(sl.lo, sl.hi);                   \
        else k_shade<false, false, false, SPEC><<<shade_grid, PB_SHADE_THREADS, shade_smem, s>>>PB_SHADE_ARGS(sl.lo, sl.hi);                                \
        launches++;                                                                                                                                       \
    } while (0)
                    case 1 + LOBE_SPEC_REFL: PB_SHADE_SOBOL_ONLY(1 + LOBE_SPEC_REFL); break;
                    case 1 + LOBE_FRESNEL_SPEC: PB_SHADE_SOBOL_ONLY(1 + LOBE_FRESNEL_SPEC); break;
                    case 1 + LOBE_OREN_NAYAR: PB_SHADE_SOBOL_ONLY(1 + LOBE_OREN_NAYAR); break;
                    case 1 + LOBE_MF_REFL: PB_SHADE_SOBOL_ONLY(1 + LOBE_MF_REFL); break;
                    case 1 + LOBE_FRESNEL_BLEND: PB_SHADE_SOBOL_ONLY(1 + LOBE_FRESNEL_BLEND); break;
                    case PB_SPEC_PLASTIC: PB_SHADE_SOBOL_ONLY(PB_SPEC_PLASTIC); break;
#undef PB_SHADE_SOBOL_ONLY
                    default: PB_SHADE_LAUNCH(0, shade_grid, sl.lo, sl.hi); break;
                }
            }
#undef PB_SHADE_LAUNCH
#undef PB_SHADE_ARGS
            CK(cudaEventRecord(f, s));
            sev.push_back(e); sev.push_back(f);
            V.cur ^= 1;
            return PBRT_OK;
        };
        auto enqueue_begin = [&](int c, const BatchInfo& bi) -> int {
            BatchCtx& X = scr->ctx[c];
            Live& V = live[c];
            V.cur = 0;
            V.iter = 0;
            uint32_t n = bi.n_pixels * bi.n_samples;
            // ray count, ray cursor, both sets of class counts (and the voxel requests): from here on the kernels reset them for each other
            CK(cudaMemsetAsync(V.d_nrays, 0, (5 + 2 * PB_SHADE_CLASSES) * sizeof(uint32_t), V.s));
            if (spatial) CK(cudaMemsetAsync(V.grid.n_request, 0, 4, V.s));
            const auto raygen = sc->cam_motion ? k_raygen<true> : k_raygen<false>;
            raygen<<<(n + 255) / 256, 256, 0, V.s>>>(sc->d, rp, V.ps, bi, sc->nib.p, n_chunks, sc->vdc.p, sc->vdci.p, X.queue[0].p, V.counts, X.rays.p, V.d_nrays,
                                                      sc->counters.p, sc->cam_mo);
            launches++;
            return PBRT_OK;
        };
        auto enqueue_end = [&](int c, const BatchInfo& bi) -> int {
            Live& V = live[c];
            k_resolve<<<(bi.n_pixels + 255) / 256, 256, 0, V.s>>>(rp, V.ps, bi, scr->filter_table.p, d_film, d_samples);
            launches++;
            return PBRT_OK;
        };

        // ---- batches ------------------------------------------------------------------------------
        std::vector<BatchInfo> batches;
        for (uint32_t s0 = 0; s0 < rp.spp; s0 += samples_per_batch)
            for (uint64_t pix0 = 0; pix0 < total_pixels; pix0 += pixels_per_batch) {
                BatchInfo bi;
                bi.first_pixel = (uint32_t)pix0;
                bi.n_pixels = (uint32_t)std::min<uint64_t>(pixels_per_batch, total_pixels - pix0);
                bi.first_sample = s0;
                bi.n_samples = std::min(samples_per_batch, rp.spp - s0);
                batches.push_back(bi);
            }
        const uint32_t iters = rp.max_depth + 1;
        int rc = PBRT_OK;
        since("setup done");
        if (null_paths) {
            // paths can pass through null surfaces without counting a bounce, so the number of iterations is only known on the
            // device.  The queue length is read one iteration late (see the DirectLighting loop): the iteration queued past the end
            // runs over empty queues, like the tail iterations of the fixed-length loop below.
            uint32_t* h_poll = nullptr;
            cudaEvent_t poll_ev[2];
            CK(scr->poll_words(&h_poll));
            CK(scr->event(&poll_ev[0])); CK(scr->event(&poll_ev[1]));
            const uint32_t lag = poll_lag();
            for (const BatchInfo& bi : batches) {
                if ((rc = enqueue_begin(0, bi)) != PBRT_OK) return rc;
                for (uint32_t it = 0;; ++it) {
                    if ((rc = enqueue_iteration(0, false)) != PBRT_OK) return rc;
                    CK(cudaMemcpyAsync(&h_poll[4u + (it & 1u)], live[0].counts + live[0].cur, 4, cudaMemcpyDeviceToHost, live[0].s));
                    CK(cudaEventRecord(poll_ev[it & 1u], live[0].s));
                    if (it >= lag) {
                        CK(cudaEventSynchronize(poll_ev[(it - lag) & 1u]));
                        if (h_poll[4u + ((it - lag) & 1u)] == 0u) break;
                    }
                }
                if ((rc = enqueue_end(0, bi)) != PBRT_OK) return rc;
            }
        } else {
            // batches are dealt to the contexts round robin; the host interleaves the two streams' launches at
            // iteration granularity so both always have work queued
            for (size_t b0 = 0; b0 < batches.size(); b0 += (size_t)n_ctx) {
                const int nb = (int)std::min<size_t>((size_t)n_ctx, batches.size() - b0);
                for (int c = 0; c < nb; ++c) if ((rc = enqueue_begin(c, batches[b0 + c])) != PBRT_OK) return rc;
                for (uint32_t it = 0; it < iters; ++it)
                    for (int c = 0; c < nb; ++c) if ((rc = enqueue_iteration(c, dual && nb >= 2 && it == 0)) != PBRT_OK) return rc;
                for (int c = 0; c < nb; ++c) if ((rc = enqueue_end(c, batches[b0 + c])) != PBRT_OK) return rc;
            }
        }
        CK(cudaGetLastError());
        since("all batches enqueued");
        // join the side streams back into the caller's stream
        if (dual)
            for (int c = 0; c < n_ctx; ++c) {
                cudaEvent_t done;
                CK(scr->event(&done));
                CK(cudaEventRecord(done, live[c].s));
                CK(cudaStreamWaitEvent(st, done, 0));
            }
        uint32_t err = 0, err1 = 0, errs[4] = {0, 0, 0, 0}, grid_full[4] = {0, 0, 0, 0};
        for (int c = 0; c < n_ctx; ++c) CK(cudaMemcpyAsync(&errs[c], live[c].d_err, 4, cudaMemcpyDeviceToHost, st));
        if (grid_sparse)
            for (int c = 0; c < n_ctx; ++c) CK(cudaMemcpyAsync(&grid_full[c], live[c].grid.n_request + 2, 4, cudaMemcpyDeviceToHost, st));
        CK(cudaEventRecord(ev1, st));
        CK(cudaStreamSynchronize(st));
        since("final sync");
        if (grid_full[0] | grid_full[1] | grid_full[2] | grid_full[3])
            return fail(PBRT_E_UNSUPPORTED, "spatial light distribution: the paths touch more voxels than the table budget holds (PB_LIGHTGRID_BYTES, "
                                            "default 4 GiB per stream context); render with the power or uniform light strategy");
        err = errs[0] | errs[1] | errs[2] | errs[3];
        if (err | err1) return fail(PBRT_E_UNSUPPORTED, halton ? "HaltonSampler can only sample 1000 dimensions (halton.rs:256-262)"
                                                               : "SobolSampler can only sample up to 1024 dimensions (sobol.rs:119-124)");
    } else {
        CK(cudaEventRecord(ev1, st));
        CK(cudaStreamSynchronize(st));
    }
    g_launches += launches;
    if (stats) {
        std::memset(stats, 0, sizeof *stats);
        DCounters c;
        CK(cudaMemcpy(&c, sc->counters.p, sizeof c, cudaMemcpyDeviceToHost));
        stats->camera_rays = c.camera_rays; stats->closest_rays = c.closest_rays; stats->shadow_rays = c.shadow_rays;
        stats->rays = c.closest_rays + c.shadow_rays;
        stats->nodes_visited = c.nodes_visited; stats->tris_tested = c.tris_tested; stats->light_tri_tests = c.light_tri_tests;
        stats->shade_slots = c.shade_slots; stats->shaded_vertices = c.shaded_vertices;
        float ms = 0.0f;
        CK(cudaEventElapsedTime(&ms, ev0, ev1));
        stats->ms_total = ms;
        for (size_t i = 0; i + 1 < tev.size(); i += 2) { float m = 0; cudaEventElapsedTime(&m, tev[i], tev[i + 1]); stats->ms_trace += m; }
        for (size_t i = 0; i + 1 < sev.size(); i += 2) { float m = 0; cudaEventElapsedTime(&m, sev[i], sev[i + 1]); stats->ms_shade += m; }
        stats->trace_launches = trace_launches;
        stats->kernel_launches = launches;
    }
    since("stats + event teardown");
    return PBRT_OK;
}

extern "C" {

int pbrt_gpu_render_device(PbrtScene* scene, const PbrtRenderParams* params, const int32_t pixel_rect[4], float* d_film_rgbw, void* cuda_stream,
                           PbrtStats* stats) {
    if (!d_film_rgbw) return fail(PBRT_E_INVALID, "null film");
    Share sh;
    sh.rect = pixel_rect;
    return render_impl(scene, params, sh, d_film_rgbw, nullptr, (cudaStream_t)cuda_stream, stats);
}

// Host-film epilogue shared by pbrt_gpu_render and pbrt_gpu_render_multi: device film -> pinned staging -> `+=` into the caller's array
static int film_to_host(DeviceScratch* scr, size_t n_floats, float* film_rgbw) {
    CK(scr->host_film(n_floats));
    CK(cudaMemcpyAsync(scr->h_film, scr->film.p, n_floats * sizeof(float), cudaMemcpyDeviceToHost, 0));
    CK(cudaStreamSynchronize(0));
    const float* src = scr->h_film;
    const unsigned nt = n_floats >= (1u << 20) ? std::max(1u, std::min(8u, std::thread::hardware_concurrency())) : 1u;
    if (nt == 1) { for (size_t i = 0; i < n_floats; ++i) film_rgbw[i] += src[i]; return PBRT_OK; }
    std::vector<std::thread> th;
    for (unsigned t = 0; t < nt; ++t)
        th.emplace_back([=] { for (size_t i = n_floats * t / nt, e = n_floats * (t + 1) / nt; i < e; ++i) film_rgbw[i] += src[i]; });
    for (auto& x : th) x.join();
    return PBRT_OK;
}

int pbrt_gpu_render(PbrtScene* scene, const PbrtRenderParams* params, const int32_t pixel_rect[4], float* film_rgbw, PbrtStats* stats) {
    if (!scene || !params || !film_rgbw) return fail(PBRT_E_INVALID, "null argument");
    CK(cudaSetDevice(scene->device));
    DeviceScratch* scr = scratch_for(scene->device);
    if (!scr) return fail(PBRT_E_INVALID, "device ordinal out of range");
    std::lock_guard<std::mutex> film_lock(scr->film_mu);
    const int32_t* cb = params->cropped_pixel_bounds;
    size_t npx = (size_t)std::max(0, cb[2] - cb[0]) * (size_t)std::max(0, cb[3] - cb[1]);
    CK(scr->film.alloc(npx * 4));
    CK(cudaMemsetAsync(scr->film.p, 0, npx * 16, 0));
    Share sh;
    sh.rect = pixel_rect;
    int rc = render_impl(scene, params, sh, scr->film.p, nullptr, 0, stats);
    if (rc != PBRT_OK) return rc;
    return film_to_host(scr, npx * 4, film_rgbw);
}

int pbrt_gpu_render_tiles_device(PbrtScene* scene, const PbrtRenderParams* params, uint32_t part, uint32_t n_parts, float* d_film_rgbw, void* cuda_stream,
                                 PbrtStats* stats) {
    if (!d_film_rgbw) return fail(PBRT_E_INVALID, "null film");
    if (n_parts == 0) return fail(PBRT_E_INVALID, "n_parts must be positive");
    Share sh;
    sh.part = part; sh.n_parts = n_parts;
    return render_impl(scene, params, sh, d_film_rgbw, nullptr, (cudaStream_t)cuda_stream, stats);
}

int pbrt_gpu_render_multi(PbrtScene* const* scenes, uint32_t n_scenes, const PbrtRenderParams* params, float* film_rgbw, PbrtStats* stats) {
    if (!scenes || n_scenes == 0 || !params || !film_rgbw) return fail(PBRT_E_INVALID, "null argument");
    if (n_scenes > 16) return fail(PBRT_E_UNSUPPORTED, "more than 16 devices");
    for (uint32_t i = 0; i < n_scenes; ++i) {
        if (!scenes[i]) return fail(PBRT_E_INVALID, "null scene");
        for (uint32_t j = 0; j < i; ++j)
            if (scenes[j]->device == scenes[i]->device) return fail(PBRT_E_INVALID, "pbrt_gpu_render_multi needs one scene per device");
    }
    const int32_t* cb = params->cropped_pixel_bounds;
    const size_t npx = (size_t)std::max(0, cb[2] - cb[0]) * (size_t)std::max(0, cb[3] - cb[1]);
    std::vector<DeviceScratch*> scr(n_scenes);
    for (uint32_t i = 0; i < n_scenes; ++i)
        if (!(scr[i] = scratch_for(scenes[i]->device))) return fail(PBRT_E_INVALID, "device ordinal out of range");
    // film locks in device order (two concurrent multi-device calls cannot deadlock)
    std::vector<uint32_t> order(n_scenes);
    for (uint32_t i = 0; i < n_scenes; ++i) order[i] = i;
    std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return scenes[a]->device < scenes[b]->device; });
    std::vector<std::unique_lock<std::mutex>> locks;
    for (uint32_t i : order) locks.emplace_back(scr[i]->film_mu);
    // ---- one host thread per device renders its share of the Morton-ordered tiles into that device's film --------------------------
    std::vector<int> rcs(n_scenes, PBRT_OK);
    std::vector<std::string> errs(n_scenes);
    std::vector<PbrtStats> sts(n_scenes);
    auto worker = [&](uint32_t i) {
        auto body = [&]() -> int {
            CK(cudaSetDevice(scenes[i]->device));
            CK(scr[i]->film.alloc(npx * 4));
            CK(cudaMemsetAsync(scr[i]->film.p, 0, npx * 16, 0));
            Share sh;
            sh.part = i; sh.n_parts = n_scenes;
            return render_impl(scenes[i], params, sh, scr[i]->film.p, nullptr, 0, &sts[i]);
        };
        rcs[i] = body();
        if (rcs[i] != PBRT_OK) errs[i] = g_err;  // g_err is thread local: carry the text back to the caller's thread
    };
    if (n_scenes == 1) worker(0);
    else {
        std::vector<std::thread> th;
        for (uint32_t i = 0; i < n_scenes; ++i) th.emplace_back(worker, i);
        for (auto& t : th) t.join();
    }
    for (uint32_t i = 0; i < n_scenes; ++i)
        if (rcs[i] != PBRT_OK) return fail(rcs[i], "device " + std::to_string(scenes[i]->device) + ": " + errs[i]);
    // ---- the single reduce of the films (SURVEY 8e): device 0 of the list sums its peers' films over NVLink peer access; a pair without
    // peer access goes through a staged copy.  A sum, not a gather: filter footprints cross tile borders (film.rs:362-367).
    const int root = scenes[0]->device;
    CK(cudaSetDevice(root));
    cudaEvent_t r0, r1;
    CK(cudaEventCreate(&r0)); CK(cudaEventCreate(&r1));
    CK(cudaEventRecord(r0, 0));
    PeerFilms direct;
    direct.n = 0;
    DevBuf<float> staged;
    for (uint32_t i = 1; i < n_scenes && npx; ++i) {
        int can = 0;
        CK(cudaDeviceCanAccessPeer(&can, root, scenes[i]->device));
        if (can) {
            cudaError_t e = cudaDeviceEnablePeerAccess(scenes[i]->device, 0);
            if (e == cudaErrorPeerAccessAlreadyEnabled) { cudaGetLastError(); e = cudaSuccess; }
            if (e != cudaSuccess) can = 0;
        }
        if (can) direct.p[direct.n++] = reinterpret_cast<const float4*>(scr[i]->film.p);
        else {
            CK(staged.alloc(npx * 4));
            CK(cudaMemcpyPeerAsync(staged.p, root, scr[i]->film.p, scenes[i]->device, npx * 16, 0));
            PeerFilms one;
            one.n = 1; one.p[0] = reinterpret_cast<const float4*>(staged.p);
            k_film_sum_peers<<<sm_count_of(root) * 4, 256>>>(reinterpret_cast<float4*>(scr[0]->film.p), one, npx);
            g_launches++;
        }
    }
    if (direct.n) {
        k_film_sum_peers<<<sm_count_of(root) * 4, 256>>>(reinterpret_cast<float4*>(scr[0]->film.p), direct, npx);
        g_launches++;
    }
    CK(cudaEventRecord(r1, 0));
    CK(cudaGetLastError());
    int rc = film_to_host(scr[0], npx * 4, film_rgbw);
    float reduce_ms = 0.0f;
    cudaEventElapsedTime(&reduce_ms, r0, r1);
    cudaEventDestroy(r0); cudaEventDestroy(r1);
    if (rc != PBRT_OK) return rc;
    if (stats) {
        std::memset(stats, 0, sizeof *stats);
        for (const PbrtStats& t : sts) {
            stats->camera_rays += t.camera_rays; stats->rays += t.rays; stats->closest_rays += t.closest_rays; stats->shadow_rays += t.shadow_rays;
            stats->nodes_visited += t.nodes_visited; stats->tris_tested += t.tris_tested; stats->light_tri_tests += t.light_tri_tests;
            stats->shade_slots += t.shade_slots; stats->shaded_vertices += t.shaded_vertices;
            stats->trace_launches += t.trace_launches; stats->kernel_launches += t.kernel_launches;
            stats->ms_total = std::max(stats->ms_total, t.ms_total);  // the devices run concurrently: the slowest one bounds the frame
            stats->ms_trace = std::max(stats->ms_trace, t.ms_trace);
            stats->ms_shade = std::max(stats->ms_shade, t.ms_shade);
        }
        stats->ms_total += reduce_ms;
    }
    return PBRT_OK;
}

int pbrt_gpu_render_samples(PbrtScene* scene, const PbrtRenderParams* params, const int32_t pixel_rect[4], float* sample_rgb, PbrtStats* stats) {
    if (!scene || !params || !sample_rgb || !pixel_rect) return fail(PBRT_E_INVALID, "null argument");
    CK(cudaSetDevice(scene->device));
    const int32_t* cb = params->cropped_pixel_bounds;
    size_t npx = (size_t)std::max(0, cb[2] - cb[0]) * (size_t)std::max(0, cb[3] - cb[1]);
    size_t ns = (size_t)std::max(0, pixel_rect[2] - pixel_rect[0]) * (size_t)std::max(0, pixel_rect[3] - pixel_rect[1]) * params->spp * 3;
    CK(scene->film.alloc(std::max<size_t>(npx * 4, 4)));
    CK(cudaMemset(scene->film.p, 0, std::max<size_t>(npx * 16, 16)));
    CK(scene->samples.alloc(std::max<size_t>(ns, 1)));
    CK(cudaMemset(scene->samples.p, 0, std::max<size_t>(ns, 1) * 4));
    Share sh;
    sh.rect = pixel_rect;
    int rc = render_impl(scene, params, sh, scene->film.p, scene->samples.p, 0, stats);
    if (rc != PBRT_OK) return rc;
    CK(cudaMemcpy(sample_rgb, scene->samples.p, ns * 4, cudaMemcpyDeviceToHost));
    return PBRT_OK;
}

static int rays_common(PbrtScene* sc, uint32_t n, const float* o, const float* d, const float* t_max, DevBuf<float>& bo, DevBuf<float>& bd,
                       DevBuf<float>& bt) {
    CK(cudaSetDevice(sc->device));
    CK(bo.alloc(3 * (size_t)n + 1)); CK(bd.alloc(3 * (size_t)n + 1)); CK(bt.alloc((size_t)n + 1));
    CK(cudaMemcpy(bo.p, o, 3 * (size_t)n * 4, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(bd.p, d, 3 * (size_t)n * 4, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(bt.p, t_max, (size_t)n * 4, cudaMemcpyHostToDevice));
    CK(sc->counters.alloc(1));
    CK(cudaMemset(sc->counters.p, 0, sizeof(DCounters)));
    if (sc->d.mesh_alpha) {  // the alpha test walks a texture graph: stack frames above the default limit (see render_impl)
        size_t cur = 0;
        CK(cudaDeviceGetLimit(&cur, cudaLimitStackSize));
        if (cur < 4096) CK(cudaDeviceSetLimit(cudaLimitStackSize, 4096));
    }
    return PBRT_OK;
}
static int rays_stats(PbrtScene* sc, PbrtStats* stats, float ms) {
    if (!stats) return PBRT_OK;
    std::memset(stats, 0, sizeof *stats);
    DCounters c;
    CK(cudaMemcpy(&c, sc->counters.p, sizeof c, cudaMemcpyDeviceToHost));
    stats->closest_rays = c.closest_rays; stats->shadow_rays = c.shadow_rays; stats->rays = c.closest_rays + c.shadow_rays;
    stats->nodes_visited = c.nodes_visited; stats->tris_tested = c.tris_tested;
    stats->ms_total = stats->ms_trace = ms;
    stats->trace_launches = stats->kernel_launches = 1;
    return PBRT_OK;
}

int pbrt_gpu_intersect(PbrtScene* sc, uint32_t n, const float* o, const float* d, const float* t_max, int32_t* prim, float* t, float* b,
                       PbrtStats* stats) {
    if (!sc || (n && (!o || !d || !t_max || !prim || !t || !b))) return fail(PBRT_E_INVALID, "null argument");
    if (n == 0) { if (stats) std::memset(stats, 0, sizeof *stats); return PBRT_OK; }
    DevBuf<float> bo, bd, bt, dt, db;
    DevBuf<int> dp;
    int rc = rays_common(sc, n, o, d, t_max, bo, bd, bt);
    if (rc != PBRT_OK) return rc;
    CK(dp.alloc(n)); CK(dt.alloc(n)); CK(db.alloc(3 * (size_t)n));
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    int grid = (int)std::min<uint64_t>(((uint64_t)n + PB_TRACE_THREADS - 1) / PB_TRACE_THREADS, (uint64_t)sm_count_of(sc->device) * 16);
    CK(cudaEventRecord(e0));
    DevBuf<uint32_t> cursor;
    CK(cursor.alloc(1));
    CK(cudaMemset(cursor.p, 0, 4));
    TraceIO io;
    std::memset(&io, 0, sizeof io);
    io.o = bo.p; io.d = bd.p; io.tmax = bt.p; io.out_prim = dp.p; io.out_t = dt.p; io.out_b = db.p;
    // instanced scenes: PBRT_INSTANCING_REFERENCE semantics (the ray-cast entry points carry no render parameters)
    if (sc->d.mesh_alpha) {
        if (sc->d.n_instances) k_trace<true, 1, false, true, true><<<grid, PB_TRACE_THREADS>>>(sc->d, io, nullptr, n, cursor.p, sc->counters.p);
        else k_trace<true, 1, false, false, true><<<grid, PB_TRACE_THREADS>>>(sc->d, io, nullptr, n, cursor.p, sc->counters.p);
    } else if (sc->d.n_instances) k_trace<true, 1, false, true><<<grid, PB_TRACE_THREADS>>>(sc->d, io, nullptr, n, cursor.p, sc->counters.p);
    else k_trace<true, 1, false><<<grid, PB_TRACE_THREADS>>>(sc->d, io, nullptr, n, cursor.p, sc->counters.p);
    CK(cudaEventRecord(e1));
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    g_launches++;
    float ms = 0;
    cudaEventElapsedTime(&ms, e0, e1);
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    CK(cudaMemcpy(prim, dp.p, (size_t)n * 4, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(t, dt.p, (size_t)n * 4, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(b, db.p, 3 * (size_t)n * 4, cudaMemcpyDeviceToHost));
    return rays_stats(sc, stats, ms);
}

int pbrt_gpu_intersect_p(PbrtScene* sc, uint32_t n, const float* o, const float* d, const float* t_max, uint8_t* occluded, PbrtStats* stats) {
    if (!sc || (n && (!o || !d || !t_max || !occluded))) return fail(PBRT_E_INVALID, "null argument");
    if (n == 0) { if (stats) std::memset(stats, 0, sizeof *stats); return PBRT_OK; }
    DevBuf<float> bo, bd, bt;
    DevBuf<unsigned char> docc;
    int rc = rays_common(sc, n, o, d, t_max, bo, bd, bt);
    if (rc != PBRT_OK) return rc;
    CK(docc.alloc(n));
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    int grid = (int)std::min<uint64_t>(((uint64_t)n + PB_TRACE_THREADS - 1) / PB_TRACE_THREADS, (uint64_t)sm_count_of(sc->device) * 16);
    CK(cudaEventRecord(e0));
    DevBuf<uint32_t> cursor;
    CK(cursor.alloc(1));
    CK(cudaMemset(cursor.p, 0, 4));
    TraceIO io;
    std::memset(&io, 0, sizeof io);
    io.o = bo.p; io.d = bd.p; io.tmax = bt.p; io.out_occ = docc.p;
    if (sc->d.mesh_alpha) {
        if (sc->d.n_instances) k_trace<true, 2, false, true, true><<<grid, PB_TRACE_THREADS>>>(sc->d, io, nullptr, n, cursor.p, sc->counters.p);
        else k_trace<true, 2, false, false, true><<<grid, PB_TRACE_THREADS>>>(sc->d, io, nullptr, n, cursor.p, sc->counters.p);
    } else if (sc->d.n_instances) k_trace<true, 2, false, true><<<grid, PB_TRACE_THREADS>>>(sc->d, io, nullptr, n, cursor.p, sc->counters.p);
    else k_trace<true, 2, false><<<grid, PB_TRACE_THREADS>>>(sc->d, io, nullptr, n, cursor.p, sc->counters.p);
    CK(cudaEventRecord(e1));
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    g_launches++;
    float ms = 0;
    cudaEventElapsedTime(&ms, e0, e1);
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    CK(cudaMemcpy(occluded, docc.p, n, cudaMemcpyDeviceToHost));
    return rays_stats(sc, stats, ms);
}

// Known-answer hook: the device's sin/cos (pb_math.cuh) for n arguments, so that tests can hold them against the host libm the
// reference calls.  Not part of the render path.
int pbrt_gpu_kat_sincos(int device, uint32_t n, const float* x, float* s_out, float* c_out) {
    if (n && (!x || !s_out || !c_out)) return fail(PBRT_E_INVALID, "null argument");
    int rc = check_device(device);
    if (rc != PBRT_OK) return rc;
    if (n == 0) return PBRT_OK;
    DevBuf<float> dx, ds, dc;
    CK(dx.alloc(n)); CK(ds.alloc(n)); CK(dc.alloc(n));
    CK(cudaMemcpy(dx.p, x, (size_t)n * 4, cudaMemcpyHostToDevice));
    k_kat_sincos<<<(n + 255) / 256, 256>>>(dx.p, n, ds.p, dc.p);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    g_launches++;
    CK(cudaMemcpy(s_out, ds.p, (size_t)n * 4, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(c_out, dc.p, (size_t)n * 4, cudaMemcpyDeviceToHost));
    return PBRT_OK;
}

// Known-answer hook: the device's acos(x[i]) and atan2(y[i], x[i]) (restatements of glibc's acosf / atan2f, pb_math.cuh)
int pbrt_gpu_kat_acos_atan2(int device, uint32_t n, const float* x, const float* y, float* acos_out, float* atan2_out) {
    if (n && (!x || !y || !acos_out || !atan2_out)) return fail(PBRT_E_INVALID, "null argument");
    int rc = check_device(device);
    if (rc != PBRT_OK) return rc;
    if (n == 0) return PBRT_OK;
    DevBuf<float> dx, dy, da, dt;
    CK(dx.alloc(n)); CK(dy.alloc(n)); CK(da.alloc(n)); CK(dt.alloc(n));
    CK(cudaMemcpy(dx.p, x, (size_t)n * 4, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(dy.p, y, (size_t)n * 4, cudaMemcpyHostToDevice));
    k_kat_acos_atan2<<<(n + 255) / 256, 256>>>(dx.p, dy.p, n, da.p, dt.p);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    g_launches++;
    CK(cudaMemcpy(acos_out, da.p, (size_t)n * 4, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(atan2_out, dt.p, (size_t)n * 4, cudaMemcpyDeviceToHost));
    return PBRT_OK;
}

// Known-answer hook: AnimatedTransform::new on the host (pb_motion.cuh), AnimatedTransform::interpolate on the device at n times.
int pbrt_gpu_kat_animated_interpolate(int device, const PbrtAnimatedTransform* at, uint32_t n, const float* times, float* m_out, float* m_inv_out) {
    if (!at || (n && (!times || !m_out || !m_inv_out))) return fail(PBRT_E_INVALID, "null argument");
    int rc = check_device(device);
    if (rc != PBRT_OK) return rc;
    if (n == 0) return PBRT_OK;
    DMotion mo;
    std::memset(&mo, 0, sizeof mo);
    motion_create(at->start, at->start_inv, at->start_time, at->end, at->end_inv, at->end_time, mo);
    DevBuf<float> dt, dm, dmi;
    CK(dt.alloc(n)); CK(dm.alloc(16 * (size_t)n)); CK(dmi.alloc(16 * (size_t)n));
    CK(cudaMemcpy(dt.p, times, (size_t)n * 4, cudaMemcpyHostToDevice));
    k_kat_motion<<<(n + 255) / 256, 256>>>(mo, dt.p, n, dm.p, dmi.p);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    g_launches++;
    CK(cudaMemcpy(m_out, dm.p, (size_t)n * 64, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(m_inv_out, dmi.p, (size_t)n * 64, cudaMemcpyDeviceToHost));
    return PBRT_OK;
}

int pbrt_gpu_kat_log2(int device, uint32_t n, const float* x, float* log2_out) {
    if (n && (!x || !log2_out)) return fail(PBRT_E_INVALID, "null argument");
    int rc = check_device(device);
    if (rc != PBRT_OK) return rc;
    if (n == 0) return PBRT_OK;
    DevBuf<float> dx, dy;
    CK(dx.alloc(n)); CK(dy.alloc(n));
    CK(cudaMemcpy(dx.p, x, (size_t)n * 4, cudaMemcpyHostToDevice));
    k_kat_log2<<<(n + 255) / 256, 256>>>(dx.p, n, dy.p);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    g_launches++;
    CK(cudaMemcpy(log2_out, dy.p, (size_t)n * 4, cudaMemcpyDeviceToHost));
    return PBRT_OK;
}

}  // extern "C"
