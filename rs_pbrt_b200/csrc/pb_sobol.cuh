// pb_sobol.cuh -- SobolSampler (global sampler) on the device.
//   sobol_interval_to_index   src/core/lowdiscrepancy.rs:1014-1043
//   sobol_sample_float        src/core/lowdiscrepancy.rs:1053-1076
//   SobolSampler::sample_dimension / get_1d / get_2d   src/samplers/sobol.rs:125-200
//   radical_inverse           src/core/lowdiscrepancy.rs:1080-1145
// The generator matrices live in data/sobol_tables.bin (see tools/extract_sobol_tables.py).
#pragma once
#include "pb_math.cuh"
#include "pb_scene.cuh"

namespace pb {

#define PB_SOBOL_MATRIX_SIZE 52
#define PB_SOBOL_DIMS 1024

// vdc / vdci: the rows for resolution exponent m (52 u64 each)
PB_D uint64_t sobol_interval_to_index(const uint64_t* __restrict__ vdc, const uint64_t* __restrict__ vdci, uint32_t m, uint64_t frame,
                                      int px, int py) {
    if (m == 0) return 0;
    const uint32_t m2 = m << 1;
    uint64_t index = frame << m2;
    uint64_t delta = 0;
    for (int c = 0; frame > 0; frame >>= 1, ++c)
        if (frame & 1) delta ^= vdc[c];
    uint64_t b = ((uint64_t)(((uint32_t)px) << m) | (uint64_t)(int64_t)py) ^ delta;
    for (int c = 0; b > 0; b >>= 1, ++c)
        if (b & 1) index ^= vdci[c];
    return index;
}

// m32: SOBOL_MATRICES_32 (row `dim`, 52 columns).  Bit-by-bit form of sobol_sample_float, used once per
// camera sample by k_raygen.
PB_D float sobol_sample_float(const uint32_t* __restrict__ m32, uint64_t a, uint32_t dim) {
    uint32_t v = 0;
    const uint32_t* row = m32 + dim * PB_SOBOL_MATRIX_SIZE;
    uint32_t lo = (uint32_t)a, hi = (uint32_t)(a >> 32);
    while (lo) { int i = __ffs(lo) - 1; v ^= row[i]; lo &= lo - 1; }
    while (hi) { int i = __ffs(hi) - 1; v ^= row[32 + i]; hi &= hi - 1; }
    // u32 -> f32 rounds to nearest even, like Rust's `as f32`
    return fminf(__uint2float_rn(v) * 2.3283064365386963e-10f, PB_ONE_MINUS_EPSILON);
}

// Nibble tables: nib[dim][chunk][e] = XOR of the generator-matrix columns 4*chunk + j over the set bits j of
// e (built on the host from SOBOL_MATRICES_32).  XOR is associative, so
//   v = XOR_chunks nib[dim][chunk][(index >> 4*chunk) & 15]
// is bit-identical to the reference's column loop with a quarter of the memory operations and no data
// dependent loop.  k_shade stages the [dims reachable] x [chunks the index can fill] slice in shared memory.
#define PB_SOBOL_CHUNKS 13  // 52 columns / 4
struct SobolCtx {
    const uint32_t* nib;   // nibble tables (shared or global memory)
    uint32_t stride;       // chunks stored per dimension in `nib`
    uint32_t n_chunks;     // chunks needed to cover every index of this render
    uint64_t index;        // interval_sample_index
    uint32_t dim;          // next dimension
    bool overflow;         // the reference panics past 1024 dimensions (sobol.rs:119-124); we flag
};
PB_D float sobol_to_float(uint32_t v) { return fminf(__uint2float_rn(v) * 2.3283064365386963e-10f, PB_ONE_MINUS_EPSILON); }
// the raw u32 of dimension `dim` (before sobol_to_float)
PB_D uint32_t sobol_sample_nib_u32(const SobolCtx& s, uint32_t dim) {
    const uint32_t* t = s.nib + (size_t)dim * s.stride * 16u;
    uint32_t lo = (uint32_t)s.index, hi = (uint32_t)(s.index >> 32);
    uint32_t v = 0;
    const uint32_t n_lo = s.n_chunks < 8u ? s.n_chunks : 8u;
    for (uint32_t c = 0; c < n_lo; ++c) { v ^= t[c * 16u + (lo & 15u)]; lo >>= 4; }
    for (uint32_t c = 8; c < s.n_chunks; ++c) { v ^= t[c * 16u + (hi & 15u)]; hi >>= 4; }
    return v;
}
PB_D float sobol_sample_nib(const SobolCtx& s, uint32_t dim) { return sobol_to_float(sobol_sample_nib_u32(s, dim)); }
// ---- transposed nibble tables for k_shade: nibT[(chunk * 16 + e) * ds + dim] ------------------------------------------------
// A path vertex draws up to seven consecutive dimensions of ONE Sobol' index (light choice, u_light, u_scattering, the BSDF
// sample); with the dimension as the fastest index the nibble of each chunk is extracted once and the seven table words sit
// next to each other (one address, immediate offsets), instead of seven independent walks over the chunks.  `ds` is odd, so
// the 16 values of a nibble fall into different banks.
struct SobolT {
    const uint32_t* nib;   // transposed slice (shared or global memory)
    uint32_t ds;           // dimension stride (dimensions stored, rounded up to odd)
    uint32_t n_chunks;
    uint64_t index;
    uint32_t dim;
    bool overflow;
};
template <int N>
PB_D void sobolT_fill(const SobolT& s, float (&out)[N]) {  // dimensions s.dim .. s.dim+N-1; the table is padded by 8 dimensions
    uint32_t acc[N];
#pragma unroll
    for (int k = 0; k < N; ++k) acc[k] = 0u;
    const uint32_t* t = s.nib + s.dim;
    uint32_t lo = (uint32_t)s.index, hi = (uint32_t)(s.index >> 32);
    const uint32_t n_lo = s.n_chunks < 8u ? s.n_chunks : 8u;
    for (uint32_t c = 0; c < n_lo; ++c) {
        const uint32_t* r = t + (c * 16u + (lo & 15u)) * s.ds;
        lo >>= 4;
#pragma unroll
        for (int k = 0; k < N; ++k) acc[k] ^= r[k];
    }
    for (uint32_t c = 8; c < s.n_chunks; ++c) {
        const uint32_t* r = t + (c * 16u + (hi & 15u)) * s.ds;
        hi >>= 4;
#pragma unroll
        for (int k = 0; k < N; ++k) acc[k] ^= r[k];
    }
#pragma unroll
    for (int k = 0; k < N; ++k) out[k] = sobol_to_float(acc[k]);
}
// consume n dimensions: the reference panics past 1024 dimensions (sobol.rs:119-124); we flag and the values are discarded
template <bool HALTON>
PB_D bool sobolT_take(SobolT& s, uint32_t n) {  // HALTON: 1000 dimensions (halton.rs:256-262)
    if (s.dim + n > (HALTON ? 1000u : (uint32_t)PB_SOBOL_DIMS)) { s.overflow = true; return false; }
    s.dim += n;
    return true;
}

PB_D uint32_t reverse_bits_32(uint32_t n) { return __brev(n); }
PB_D uint64_t reverse_bits_64(uint64_t n) { return __brevll(n); }
PB_D float radical_inverse_specialized(uint32_t base, uint64_t a) {
    const float inv_base = 1.0f / (float)base;
    uint64_t reversed = 0;
    float inv_base_n = 1.0f;
    while (a != 0) {
        uint64_t next = a / base;
        uint64_t digit = a - next * base;
        reversed = reversed * base + digit;
        inv_base_n *= inv_base;
        a = next;
    }
    return fminf(__ull2float_rn(reversed) * inv_base_n, PB_ONE_MINUS_EPSILON);
}
PB_D float radical_inverse(int base_index, uint64_t a) {
    switch (base_index) {
        case 0: return __ull2float_rn(reverse_bits_64(a)) * 5.421010862427522e-20f;  // 0x1p-64
        case 1: return radical_inverse_specialized(3, a);
        case 2: return radical_inverse_specialized(5, a);
        case 3: return radical_inverse_specialized(7, a);
        default: return radical_inverse_specialized(11, a);
    }
}

// ---- HaltonSampler (src/samplers/halton.rs, src/core/lowdiscrepancy.rs:788-797,1101-1122) -------------------------------------
#define PB_HALTON_DIMS 1000  // PRIME_TABLE_SIZE: the reference panics beyond (halton.rs:256-262)
// inverse_radical_inverse
PB_D uint32_t inverse_radical_inverse(uint32_t base, uint32_t inverse, uint32_t n_digits) {
    uint32_t index = 0;
    for (uint32_t i = 0; i < n_digits; ++i) {
        uint32_t digit = inverse % base;
        inverse /= base;
        index = index * base + digit;
    }
    return index;
}
// HaltonSampler::get_index_for_sample: the Halton index of sample `sample_num` of pixel (px, py) (the offset the reference
// caches per pixel is a pure function of the pixel)
PB_D uint64_t halton_index(const DRender& rp, int px, int py, uint64_t sample_num) {
    uint64_t offset = 0;
    if (rp.h_stride > 1u) {
        int pmx = px - (px / 128) * 128, pmy = py - (py / 128) * 128;  // mod_t(p, K_MAX_RESOLUTION)
        if (pmx < 0) pmx += 128;
        if (pmy < 0) pmy += 128;
        offset += (uint64_t)inverse_radical_inverse(2u, (uint32_t)pmx, rp.h_exp[0]) * (uint64_t)(rp.h_stride / rp.h_scale[0]) * (uint64_t)rp.h_mult[0];
        offset += (uint64_t)inverse_radical_inverse(3u, (uint32_t)pmy, rp.h_exp[1]) * (uint64_t)(rp.h_stride / rp.h_scale[1]) * (uint64_t)rp.h_mult[1];
        offset %= (uint64_t)rp.h_stride;
    }
    return offset + sample_num * (uint64_t)rp.h_stride;
}
// scrambled_radical_inverse for a 32-bit index (the host rejects renders whose indices do not fit); a / prime through
// the precomputed ceil(2^64 / prime): exact for every a < 2^32
PB_D float halton_scrambled(const DRender& rp, uint32_t a, uint32_t dim) {
    const uint4 e = __ldg(rp.h_dims + dim);
    const uint32_t base = e.x;
    const uint16_t* __restrict__ perm = rp.h_perm + e.y;
    const uint64_t magic = ((uint64_t)e.w << 32) | e.z;
    const float inv_base = 1.0f / (float)base;
    uint64_t reversed = 0;
    float inv_base_n = 1.0f;
    while (a != 0u) {
        const uint32_t next = (uint32_t)__umul64hi((uint64_t)a, magic);
        const uint32_t digit = a - next * base;
        reversed = reversed * base + (uint64_t)__ldg(perm + digit);
        inv_base_n *= inv_base;
        a = next;
    }
    return fminf(inv_base_n * (__ull2float_rn(reversed) + inv_base * (float)__ldg(perm) / (1.0f - inv_base)), PB_ONE_MINUS_EPSILON);
}
// HaltonSampler::sample_dimension
PB_D float halton_sample_dimension(const DRender& rp, uint64_t index, uint32_t dim) {
    if (rp.h_center && dim < 2u) return 0.5f;
    if (dim == 0u) return radical_inverse(0, index >> rp.h_exp[0]);
    if (dim == 1u) return radical_inverse(1, index / (uint64_t)rp.h_scale[1]);
    return halton_scrambled(rp, (uint32_t)index, dim);
}

}  // namespace pb
