// pb_math.cuh -- f32 device math for the rs_pbrt PathIntegrator hot path on sm_90a.
//
// Arithmetic contract (DESIGN.md "Numerics"): every expression is evaluated in the same
// operation order as the reference's Rust (file:line cited per function), with IEEE
// round-to-nearest +,-,*,/,sqrt and NO fused multiply-add (the translation unit is compiled with
// -fmad=false; rustc/LLVM never contracts).  sin and cos restate glibc's sinf/cosf bit for bit (below);
// acos and atan2 (infinite lights only) restate glibc's acosf / atan2f the same way.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define PB_HD __host__ __device__ __forceinline__
#define PB_D __device__ __forceinline__
#ifdef PB_HOST_EMU
#define PB_NOINLINE __attribute__((noinline))
#else
#define PB_NOINLINE __noinline__
#endif

namespace pb {

// src/core/pbrt.rs:16-23, src/core/rng.rs:13
#define PB_MACHINE_EPSILON 5.9604644775390625e-8f
#define PB_SHADOW_EPSILON 0.0001f
#define PB_PI 3.14159265358979323846f
#define PB_INV_PI 0.31830988618379067154f
#define PB_INV_2_PI 0.15915494309189533577f
#define PB_PI_OVER_2 1.57079632679489661923f
#define PB_PI_OVER_4 0.78539816339744830961f
#define PB_TAU 6.28318530717958647692f
#define PB_ONE_MINUS_EPSILON 0.99999994f

// gamma(n) = n*eps / (1 - n*eps)   src/core/pbrt.rs:94-96   (folded at compile time: IEEE either way)
PB_HD float gamma_n(int n) { return ((float)n * PB_MACHINE_EPSILON) / (1.0f - (float)n * PB_MACHINE_EPSILON); }

struct V3 {
    float x, y, z;
};
PB_HD V3 mk3(float x, float y, float z) { V3 v; v.x = x; v.y = y; v.z = z; return v; }
PB_HD V3 operator+(V3 a, V3 b) { return mk3(a.x + b.x, a.y + b.y, a.z + b.z); }
PB_HD V3 operator-(V3 a, V3 b) { return mk3(a.x - b.x, a.y - b.y, a.z - b.z); }
PB_HD V3 operator-(V3 a) { return mk3(-a.x, -a.y, -a.z); }
PB_HD V3 operator*(V3 a, float s) { return mk3(a.x * s, a.y * s, a.z * s); }
// vector / f32 multiplies by the reciprocal (geometry.rs:1262-1291)
PB_HD V3 vdiv(V3 a, float s) { float inv = 1.0f / s; return mk3(a.x * inv, a.y * inv, a.z * inv); }
PB_HD float dot3(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }  // geometry.rs:630
PB_HD float absdot3(V3 a, V3 b) { return fabsf(dot3(a, b)); }
PB_HD float len2(V3 a) { return a.x * a.x + a.y * a.y + a.z * a.z; }
PB_HD float len3(V3 a) { return sqrtf(len2(a)); }
PB_HD V3 norm3(V3 a) { return vdiv(a, len3(a)); }  // geometry.rs:412
PB_HD V3 abs3(V3 a) { return mk3(fabsf(a.x), fabsf(a.y), fabsf(a.z)); }
PB_HD float comp(V3 a, int i) { return i == 0 ? a.x : (i == 1 ? a.y : a.z); }
// cross product in f64, rounded once (geometry.rs:680-692)
PB_HD V3 cross3(V3 a, V3 b) {
    double ax = a.x, ay = a.y, az = a.z, bx = b.x, by = b.y, bz = b.z;
    return mk3((float)((ay * bz) - (az * by)), (float)((az * bx) - (ax * bz)), (float)((ax * by) - (ay * bx)));
}
PB_HD float maxcomp(V3 v) { return fmaxf(v.x, fmaxf(v.y, v.z)); }  // geometry.rs:711
PB_HD int maxdim(V3 v) {                                           // geometry.rs:721-734
    if (v.x > v.y) return (v.x > v.z) ? 0 : 2;
    return (v.y > v.z) ? 1 : 2;
}
PB_HD V3 faceforward3(V3 n, V3 v) { return (dot3(n, v) < 0.0f) ? -n : n; }  // geometry.rs:1842-1858
PB_HD void coordinate_system(V3 v1, V3& v2, V3& v3) {                       // geometry.rs:779-794
    if (fabsf(v1.x) > fabsf(v1.y)) v2 = vdiv(mk3(-v1.z, 0.0f, v1.x), sqrtf(v1.x * v1.x + v1.z * v1.z));
    else v2 = vdiv(mk3(0.0f, v1.z, -v1.y), sqrtf(v1.y * v1.y + v1.z * v1.z));
    v3 = cross3(v1, v2);
}

PB_HD uint32_t f2u(float f) {
#ifdef __CUDA_ARCH__
    return __float_as_uint(f);
#else
    union { float f; uint32_t u; } c; c.f = f; return c.u;
#endif
}
PB_HD float u2f(uint32_t u) {
#ifdef __CUDA_ARCH__
    return __uint_as_float(u);
#else
    union { float f; uint32_t u; } c; c.u = u; return c.f;
#endif
}
// src/core/pbrt.rs:61-91
PB_HD float next_float_up(float v) {
    if (isinf(v) && v > 0.0f) return v;
    if (v == -0.0f) v = 0.0f;
    uint32_t ui = f2u(v);
    if (v >= 0.0f) ui += 1; else ui -= 1;
    return u2f(ui);
}
PB_HD float next_float_down(float v) {
    if (isinf(v) && v < 0.0f) return v;
    if (v == 0.0f) v = -0.0f;
    uint32_t ui = f2u(v);
    if (v > 0.0f) ui -= 1; else ui += 1;
    return u2f(ui);
}
// pnt3_offset_ray_origin  src/core/geometry.rs:1535-1556
PB_HD V3 offset_ray_origin(V3 p, V3 p_error, V3 n, V3 w) {
    float d = dot3(abs3(n), p_error);
    V3 off = n * d;
    if (dot3(w, n) < 0.0f) off = -off;
    V3 po = p + off;
    if (off.x > 0.0f) po.x = next_float_up(po.x); else if (off.x < 0.0f) po.x = next_float_down(po.x);
    if (off.y > 0.0f) po.y = next_float_up(po.y); else if (off.y < 0.0f) po.y = next_float_down(po.y);
    if (off.z > 0.0f) po.z = next_float_up(po.z); else if (off.z < 0.0f) po.z = next_float_down(po.z);
    return po;
}
// a / b for call sites whose numerator is very often exactly zero (an occluded light sample, a point on the world bound, a BSDF
// pdf below the horizon).  div.rn.f32 leaves its inline fast path for a zero operand and calls a ~50-instruction subroutine --
// a visible share of k_shade's dynamic instructions on the Cornell box (DESIGN.md section 9).  IEEE
// defines 0 / b for every b that is neither 0 nor NaN as a zero whose sign is sign(a) ^ sign(b); everything else takes the real
// division.  tools/checks/fdiv0_check.cpp holds this against the hardware division on the host.
PB_HD float fdiv0(float a, float b) {
    if (a == 0.0f && b != 0.0f && b == b) return u2f((f2u(a) ^ f2u(b)) & 0x80000000u);
    return a / b;
}
// Rust `x as i32`: saturating, NaN -> 0.  cvt.rzi.s32.f32 has exactly these semantics on the
// device; the host branch spells them out.
PB_HD int f2i_sat(float x) {
#ifdef __CUDA_ARCH__
    return __float2int_rz(x);
#else
    if (x != x) return 0;
    if (x >= 2147483648.0f) return 2147483647;
    if (x <= -2147483648.0f) return (-2147483647 - 1);
    return (int)x;
#endif
}
// Division by a divisor the host knows: magic_of(d) = ceil(2^64 / d) for d >= 2, and div_magic(n, magic_of(d)) == n / d for every n < 2^32
// (the rounding error n * (magic - 2^64 / d) / 2^64 < 2^-32 stays below the 1 / d that n / d lies below the next integer).  d == 1: magic 0.
PB_HD uint64_t magic_of(uint32_t d) { return d >= 2u ? ~0ull / d + 1ull : 0ull; }
PB_HD uint32_t div_magic(uint32_t n, uint64_t magic) {
    if (!magic) return n;
#ifdef __CUDA_ARCH__
    return (uint32_t)__umul64hi((unsigned long long)n, (unsigned long long)magic);
#else
    return (uint32_t)(((unsigned __int128)n * magic) >> 64);
#endif
}
PB_HD float clampf(float v, float lo, float hi) { return v < lo ? lo : (v > hi ? hi : v); }  // pbrt.rs:108-121
PB_HD float lerpf(float t, float a, float b) { return a * (1.0f - t) + b * t; }              // pbrt.rs:235-245

// f32 sin/cos exactly as the host libm computes them.  The reference calls Rust's f32::sin/cos, i.e. glibc's sinf/cosf
// (>= 2.28: sysdeps/ieee754/flt-32/s_sincosf.h -- a double-precision polynomial on x - n*pi/2, rounded once to f32; faithfully,
// not always correctly, rounded).  The routine below restates that published algorithm with the fused multiply-adds of
// glibc's FMA ifunc variant; tools/checks/glibc_sincosf_check.c compares it with libm for every float |x| < 120
// (2.2e9 values: 0 mismatches with FMA, 34 without).  |x| >= 120 falls back to the f64 functions (never reached by the path:
// its arguments are bounded by 2*pi).
struct GlibcSinCos { double x, x2; int n; bool neg_cos; int small; };  // small: 0 = polynomial, 1 = |y| < 2^-12, 2 = out of range
PB_D GlibcSinCos glibc_sincos_reduce(float y) {
    GlibcSinCos r;
    const uint32_t top = (__float_as_uint(y) >> 20) & 0x7ffu;  // abstop12
    double x = (double)y;
    r.n = 0; r.neg_cos = false; r.small = 0;
    if (top < 0x3f4u) {  // abstop12(pi/4)
        if (top < 0x398u) r.small = 1;  // abstop12(2^-12)
        r.x = x; r.x2 = x * x;
        return r;
    }
    if (top >= 0x42fu) { r.small = 2; r.x = x; r.x2 = 0.0; return r; }  // abstop12(120.0f)
    const double rr = x * 0x1.45F306DC9C883p+23;  // 2/pi * 2^24
    const int n = (__double2int_rz(rr) + 0x800000) >> 24;
    x = __fma_rn(-(double)n, 0x1.921FB54442D18p0, x);
    const double sgn = ((n + 1) & 2) ? -1.0 : 1.0;  // sign[n & 3] = {1, -1, -1, 1}
    r.n = n; r.neg_cos = (n & 2) != 0;
    r.x2 = x * x;
    r.x = x * sgn;
    return r;
}
// both polynomials of the reduced argument; sinf_poly(.., n) is the sine one for even n and the cosine one for odd n
// (computed branch-free: the lanes of a warp land in different quadrants)
PB_D void glibc_sincos_polys(const GlibcSinCos& r, float& sin_poly, float& cos_poly) {
    const double x = r.x, x2 = r.x2;
    const double x3 = x * x2;
    const double s1 = __fma_rn(x2, -0x1.994eb3774cf24p-13, 0x1.1107605230bc4p-7);
    const double x7 = x3 * x2;
    const double s = __fma_rn(x3, -0x1.555545995a603p-3, x);
    sin_poly = (float)__fma_rn(x7, s1, s);
    const double sg = r.neg_cos ? -1.0 : 1.0;  // __sincosf_table[1] holds the negated cosine polynomial
    const double x4 = x2 * x2;
    const double c2 = __fma_rn(x2, sg * 0x1.99343027bf8c3p-16, sg * -0x1.6c087e89a359dp-10);
    const double c1 = __fma_rn(x2, sg * -0x1.ffffffd0c621cp-2, sg * 1.0);
    const double x6 = x4 * x2;
    const double c = __fma_rn(x4, sg * 0x1.55553e1068f19p-5, c1);
    cos_poly = (float)__fma_rn(x6, c2, c);
}
PB_D void sincos_rn(float y, float& s, float& c) {  // one range reduction and one evaluation of each polynomial for both
    const GlibcSinCos r = glibc_sincos_reduce(y);
    if (r.small == 2) { s = (float)sin((double)y); c = (float)cos((double)y); return; }
    float sp, cp;
    glibc_sincos_polys(r, sp, cp);
    const bool odd = (r.n & 1) != 0;
    s = odd ? cp : sp;  // sinf: sinf_poly(x*sign, x*x, p, n)
    c = odd ? sp : cp;  // cosf: sinf_poly(x*sign, x*x, p, n ^ 1)
    if (r.small == 1) { s = y; c = 1.0f; }
}
PB_D float sin_rn(float y) { float s, c; sincos_rn(y, s, c); return s; }
PB_D float cos_rn(float y) { float s, c; sincos_rn(y, s, c); return c; }

// f32 acos / atan2 exactly as the host libm computes them (glibc 2.39: the fdlibm-derived single-precision routines
// sysdeps/ieee754/flt-32/{e_acosf,s_atanf,e_atan2f}.c -- plain f32 arithmetic, which -fmad=false keeps un-fused here).
// tools/checks/glibc_acosf_atan2f_check.c holds this restatement against libm: acosf on every float of [-1, 1], atanf on every
// finite float, atan2f on 9.6e8 pairs -- 0 mismatches.  Used by InfiniteAreaLight (spherical_theta / spherical_phi).
PB_D float bitsf(uint32_t u) { return __uint_as_float(u); }
PB_D float acos_rn(float x) {
    const float one = 1.0f, pi = bitsf(0x40490fdau), pio2_hi = bitsf(0x3fc90fdau), pio2_lo = bitsf(0x33a22168u);
    const float pS0 = bitsf(0x3e2aaaabu), pS1 = -bitsf(0x3ea6b090u), pS2 = bitsf(0x3e4e0aa8u), pS3 = -bitsf(0x3d241146u), pS4 = bitsf(0x3a4f7f04u),
                pS5 = bitsf(0x3811ef08u);
    const float qS1 = -bitsf(0x4019d139u), qS2 = bitsf(0x4001572du), qS3 = -bitsf(0x3f303361u), qS4 = bitsf(0x3d9dc62eu);
    const int hx = __float_as_int(x), ix = hx & 0x7fffffff;
    if (ix == 0x3f800000) return hx > 0 ? 0.0f : pi + 2.0f * pio2_lo;
    if (ix > 0x3f800000) return (x - x) / (x - x);
    float z, p, q, r, w, s, c, df;
    if (ix < 0x3f000000) {
        if (ix <= 0x32800000) return pio2_hi + pio2_lo;
        z = x * x;
        p = z * (pS0 + z * (pS1 + z * (pS2 + z * (pS3 + z * (pS4 + z * pS5)))));
        q = one + z * (qS1 + z * (qS2 + z * (qS3 + z * qS4)));
        r = p / q;
        return pio2_hi - (x - (pio2_lo - x * r));
    } else if (hx < 0) {
        z = (one + x) * 0.5f;
        p = z * (pS0 + z * (pS1 + z * (pS2 + z * (pS3 + z * (pS4 + z * pS5)))));
        q = one + z * (qS1 + z * (qS2 + z * (qS3 + z * qS4)));
        s = sqrtf(z);
        r = p / q;
        w = r * s - pio2_lo;
        return pi - 2.0f * (s + w);
    }
    z = (one - x) * 0.5f;
    s = sqrtf(z);
    df = bitsf(__float_as_uint(s) & 0xfffff000u);
    c = (z - df * df) / (s + df);
    p = z * (pS0 + z * (pS1 + z * (pS2 + z * (pS3 + z * (pS4 + z * pS5)))));
    q = one + z * (qS1 + z * (qS2 + z * (qS3 + z * qS4)));
    r = p / q;
    w = r * s + c;
    return 2.0f * (df + w);
}
PB_D float atan_rn(float x) {
    const float aT0 = bitsf(0x3eaaaaabu), aT1 = -bitsf(0x3e4ccccdu), aT2 = bitsf(0x3e124925u), aT3 = -bitsf(0x3de38e38u), aT4 = bitsf(0x3dba2e6eu),
                aT5 = -bitsf(0x3d9d8795u), aT6 = bitsf(0x3d886b35u), aT7 = -bitsf(0x3d6ef16bu), aT8 = bitsf(0x3d4bda59u), aT9 = bitsf(0xbd15a221u),
                aT10 = bitsf(0x3c8569d7u);
    const int hx = __float_as_int(x), ix = hx & 0x7fffffff;
    float hi = 0.0f, lo = 0.0f;
    bool reduced = true;
    if (ix >= 0x4c000000) {
        if (ix > 0x7f800000) return x + x;
        return hx > 0 ? bitsf(0x3fc90fdau) + bitsf(0x33a22168u) : -bitsf(0x3fc90fdau) - bitsf(0x33a22168u);
    }
    if (ix < 0x3ee00000) {
        if (ix < 0x31000000) return x;
        reduced = false;
    } else {
        x = fabsf(x);
        if (ix < 0x3f980000) {
            if (ix < 0x3f300000) { hi = bitsf(0x3eed6338u); lo = bitsf(0x31ac3769u); x = (2.0f * x - 1.0f) / (2.0f + x); }
            else { hi = bitsf(0x3f490fdau); lo = bitsf(0x33222168u); x = (x - 1.0f) / (x + 1.0f); }
        } else {
            if (ix < 0x401c0000) { hi = bitsf(0x3f7b985eu); lo = bitsf(0x33140fb4u); x = (x - 1.5f) / (1.0f + 1.5f * x); }
            else { hi = bitsf(0x3fc90fdau); lo = bitsf(0x33a22168u); x = -1.0f / x; }
        }
    }
    float z = x * x;
    const float w = z * z;
    const float s1 = z * (aT0 + w * (aT2 + w * (aT4 + w * (aT6 + w * (aT8 + w * aT10)))));
    const float s2 = w * (aT1 + w * (aT3 + w * (aT5 + w * (aT7 + w * aT9))));
    if (!reduced) return x - x * (s1 + s2);
    z = hi - ((x * (s1 + s2) - lo) - x);
    return hx < 0 ? -z : z;
}
PB_D float atan2_rn(float y, float x) {
    const float tiny = 1.0e-30f, pi_o_4 = bitsf(0x3f490fdbu), pi_o_2 = bitsf(0x3fc90fdbu), pi = bitsf(0x40490fdbu), pi_lo = -bitsf(0x33bbbd2eu);
    const int hx = __float_as_int(x), ix = hx & 0x7fffffff, hy = __float_as_int(y), iy = hy & 0x7fffffff;
    if (ix > 0x7f800000 || iy > 0x7f800000) return x + y;
    if (hx == 0x3f800000) return atan_rn(y);
    const int m = ((hy >> 31) & 1) | ((hx >> 30) & 2);
    if (iy == 0) return m < 2 ? y : (m == 2 ? pi + tiny : -pi - tiny);
    if (ix == 0) return hy < 0 ? -pi_o_2 - tiny : pi_o_2 + tiny;
    if (ix == 0x7f800000) {
        if (iy == 0x7f800000) return m == 0 ? pi_o_4 + tiny : (m == 1 ? -pi_o_4 - tiny : (m == 2 ? 3.0f * pi_o_4 + tiny : -3.0f * pi_o_4 - tiny));
        return m == 0 ? 0.0f : (m == 1 ? -0.0f : (m == 2 ? pi + tiny : -pi - tiny));
    }
    if (iy == 0x7f800000) return hy < 0 ? -pi_o_2 - tiny : pi_o_2 + tiny;
    const int k = (iy - ix) >> 23;
    float z;
    if (k > 60) z = pi_o_2 + 0.5f * pi_lo;
    else if (hx < 0 && k < -60) z = 0.0f;
    else z = atan_rn(fabsf(y / x));
    if (m == 0) return z;
    if (m == 1) return bitsf(__float_as_uint(z) ^ 0x80000000u);
    if (m == 2) return pi - (z - pi_lo);
    return (z - pi_lo) - pi;
}

// glibc 2.39 log2f (sysdeps/ieee754/flt-32/e_log2f.c; the -mfma ifunc variant, so each a*b+c of the source is fused): MIPMap level
// selection takes log2 of the filter width (mipmap.rs:236, 288).  tools/checks/glibc_log2f_check.c holds this text against the host
// libm over every non-negative float.
__device__ const double pb_log2f_tab[32] = {
    0x1.661ec79f8f3bep+0, -0x1.efec65b963019p-2, 0x1.571ed4aaf883dp+0, -0x1.b0b6832d4fca4p-2, 0x1.49539f0f010bp+0, -0x1.7418b0a1fb77bp-2,
    0x1.3c995b0b80385p+0, -0x1.39de91a6dcf7bp-2, 0x1.30d190c8864a5p+0, -0x1.01d9bf3f2b631p-2, 0x1.25e227b0b8eap+0, -0x1.97c1d1b3b7afp-3,
    0x1.1bb4a4a1a343fp+0, -0x1.2f9e393af3c9fp-3, 0x1.12358f08ae5bap+0, -0x1.960cbbf788d5cp-4, 0x1.0953f419900a7p+0, -0x1.a6f9db6475fcep-5,
    0x1p+0, 0x0p+0, 0x1.e608cfd9a47acp-1, 0x1.338ca9f24f53dp-4, 0x1.ca4b31f026aap-1, 0x1.476a9543891bap-3,
    0x1.b2036576afce6p-1, 0x1.e840b4ac4e4d2p-3, 0x1.9c2d163a1aa2dp-1, 0x1.40645f0c6651cp-2, 0x1.886e6037841edp-1, 0x1.88e9c2c1b9ff8p-2,
    0x1.767dcf5534862p-1, 0x1.ce0a44eb17bccp-2};
PB_D float log2_rn(float x) {
    uint32_t ix = __float_as_uint(x);
    if (ix == 0x3f800000u) return 0.0f;
    if (ix - 0x00800000u >= 0x7f800000u - 0x00800000u) {
        if (ix * 2u == 0u) return bitsf(0xff800000u);
        if (ix == 0x7f800000u) return x;
        if ((ix & 0x80000000u) || ix * 2u >= 0xff000000u) return bitsf(0x7fc00000u);
        ix = __float_as_uint(x * 8388608.0f);  // subnormal: normalise
        ix -= 23u << 23;
    }
    const uint32_t tmp = ix - 0x3f330000u;
    const uint32_t i = (tmp >> 19) & 15u;
    const uint32_t iz = ix - (tmp & 0xff800000u);
    const int k = (int)tmp >> 23;
    const double invc = pb_log2f_tab[2 * i], logc = pb_log2f_tab[2 * i + 1];
    const double r = __fma_rn((double)__uint_as_float(iz), invc, -1.0);
    const double y0 = logc + (double)k;
    const double r2 = r * r;
    double y = __fma_rn(0x1.ecabf496832ep-2, r, -0x1.715479ffae3dep-1);
    y = __fma_rn(-0x1.712b6f70a7e4dp-2, r2, y);
    const double p = __fma_rn(0x1.715475f35c8b8p0, r, y0);
    return (float)__fma_rn(y, r2, p);
}

// glibc 2.39 logf (sysdeps/ieee754/flt-32/e_logf.c, -mfma ifunc variant): roughness_to_alpha of a textured roughness
// (microfacet.rs:243-255).  tools/checks/glibc_logf_check.c: 0 mismatches against the host libm over every non-negative float.
__device__ const double pb_logf_tab[32] = {
    0x1.661ec79f8f3bep+0, -0x1.57bf7808caadep-2, 0x1.571ed4aaf883dp+0, -0x1.2bef0a7c06ddbp-2, 0x1.49539f0f010bp+0, -0x1.01eae7f513a67p-2,
    0x1.3c995b0b80385p+0, -0x1.b31d8a68224e9p-3, 0x1.30d190c8864a5p+0, -0x1.6574f0ac07758p-3, 0x1.25e227b0b8eap+0, -0x1.1aa2bc79c81p-3,
    0x1.1bb4a4a1a343fp+0, -0x1.a4e76ce8c0e5ep-4, 0x1.12358f08ae5bap+0, -0x1.1973c5a611cccp-4, 0x1.0953f419900a7p+0, -0x1.252f438e10c1ep-5,
    0x1p+0, 0x0p+0, 0x1.e608cfd9a47acp-1, 0x1.aa5aa5df25984p-5, 0x1.ca4b31f026aap-1, 0x1.c5e53aa362eb4p-4,
    0x1.b2036576afce6p-1, 0x1.526e57720db08p-3, 0x1.9c2d163a1aa2dp-1, 0x1.bc2860d22477p-3, 0x1.886e6037841edp-1, 0x1.1058bc8a07ee1p-2,
    0x1.767dcf5534862p-1, 0x1.4043057b6ee09p-2};
PB_D float log_rn(float x) {
    uint32_t ix = __float_as_uint(x);
    if (ix == 0x3f800000u) return 0.0f;
    if (ix - 0x00800000u >= 0x7f800000u - 0x00800000u) {
        if (ix * 2u == 0u) return bitsf(0xff800000u);
        if (ix == 0x7f800000u) return x;
        if ((ix & 0x80000000u) || ix * 2u >= 0xff000000u) return bitsf(0x7fc00000u);
        ix = __float_as_uint(x * 8388608.0f);
        ix -= 23u << 23;
    }
    const uint32_t tmp = ix - 0x3f330000u;
    const uint32_t i = (tmp >> 19) & 15u;
    const int k = (int)tmp >> 23;
    const uint32_t iz = ix - (tmp & 0xff800000u);
    const double invc = pb_logf_tab[2 * i], logc = pb_logf_tab[2 * i + 1];
    const double r = __fma_rn((double)__uint_as_float(iz), invc, -1.0);
    const double y0 = __fma_rn((double)k, 0x1.62e42fefa39efp-1, logc);
    const double r2 = r * r;
    double y = __fma_rn(0x1.5575b0be00b6ap-2, r, -0x1.ffffef20a4123p-2);
    y = __fma_rn(-0x1.00ea348b88334p-2, r2, y);
    return (float)__fma_rn(y, r2, y0 + r);
}

// RGBSpectrum (src/core/spectrum.rs:1530-1780)
struct Sp {
    float r, g, b;
};
PB_HD Sp mksp(float r, float g, float b) { Sp s; s.r = r; s.g = g; s.b = b; return s; }
PB_HD Sp sp1(float v) { return mksp(v, v, v); }
PB_HD Sp operator+(Sp a, Sp b) { return mksp(a.r + b.r, a.g + b.g, a.b + b.b); }
PB_HD Sp operator-(Sp a, Sp b) { return mksp(a.r - b.r, a.g - b.g, a.b - b.b); }
PB_HD Sp operator*(Sp a, Sp b) { return mksp(a.r * b.r, a.g * b.g, a.b * b.b); }
PB_HD Sp operator/(Sp a, Sp b) { return mksp(a.r / b.r, a.g / b.g, a.b / b.b); }
PB_HD Sp operator*(Sp a, float s) { return mksp(a.r * s, a.g * s, a.b * s); }
PB_HD Sp operator/(Sp a, float s) { return mksp(a.r / s, a.g / s, a.b / s); }  // true division (spectrum.rs:1752)
PB_HD bool is_black(Sp a) { return a.r == 0.0f && a.g == 0.0f && a.b == 0.0f; }
PB_HD bool has_nans(Sp a) { return a.r != a.r || a.g != a.g || a.b != a.b; }
PB_HD float lum(Sp a) { return 0.212671f * a.r + 0.715160f * a.g + 0.072169f * a.b; }  // spectrum.rs:1581
PB_HD float maxsp(Sp a) { return fmaxf(fmaxf(a.r, a.g), a.b); }
PB_HD Sp sqrtsp(Sp a) { return mksp(sqrtf(a.r), sqrtf(a.g), sqrtf(a.b)); }
PB_HD Sp spdiv0(Sp a, float s) { return mksp(fdiv0(a.r, s), fdiv0(a.g, s), fdiv0(a.b, s)); }  // operator/ for often-black numerators

}  // namespace pb
