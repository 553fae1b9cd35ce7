// pb_motion.cuh -- two-keyframe AnimatedTransform (src/core/transform.rs:893-940, 2032-2124; src/core/quaternion.rs).
//
// The library decomposes each keyframe once, on the host, when the scene is created (motion_create); the kernels interpolate at the
// ray's time (motion_interpolate).  Both restate the reference in its own operation order, so that an interpolated transform is
// bit-identical to the one rs_pbrt builds: f32 throughout, glibc's acosf / sinf / cosf through their device restatements.
#pragma once
#include "pb_math.cuh"

namespace pb {

struct DQuat { float x, y, z, w; };  // Quaternion {v, w}

// AnimatedTransform::new's state minus the motion-derivative terms (which only motion_bounds reads).  Matrices are row-major 4x4.
struct DMotion {
    float start[16], start_inv[16], end[16], end_inv[16];
    float start_time, end_time;
    uint32_t actually_animated, has_rotation;
    float t[2][3];   // translations
    DQuat r[2];      // rotations (r[1] flipped onto r[0]'s hemisphere)
    float s[2][9];   // upper 3x3 of the scale matrices (the rest of S is the identity's)
};

// mtx_mul (transform.rs:238-249)
PB_HD void mx_mul(const float* a, const float* b, float* out) {
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j)
            out[4 * i + j] = a[4 * i] * b[j] + a[4 * i + 1] * b[4 + j] + a[4 * i + 2] * b[8 + j] + a[4 * i + 3] * b[12 + j];
}
// Matrix4x4::inverse (transform.rs:128-201): Gauss-Jordan with full pivoting, in place on a copy
PB_HD void mx_inverse(const float* m, float* out) {
    int indxc[4] = {0, 0, 0, 0}, indxr[4] = {0, 0, 0, 0}, ipiv[4] = {0, 0, 0, 0};
    float minv[16];
    for (int k = 0; k < 16; ++k) minv[k] = m[k];
    for (int i = 0; i < 4; ++i) {
        int irow = 0, icol = 0;
        float big = 0.0f;
        for (int j = 0; j < 4; ++j)
            if (ipiv[j] != 1)
                for (int k = 0; k < 4; ++k)
                    if (ipiv[k] == 0) {
                        const float a = fabsf(minv[4 * j + k]);
                        if (a >= big) { big = a; irow = j; icol = k; }
                    }
        ++ipiv[icol];
        if (irow != icol)
            for (int k = 0; k < 4; ++k) { const float sw = minv[4 * irow + k]; minv[4 * irow + k] = minv[4 * icol + k]; minv[4 * icol + k] = sw; }
        indxr[i] = irow; indxc[i] = icol;
        const float pivinv = 1.0f / minv[4 * icol + icol];
        minv[4 * icol + icol] = 1.0f;
        for (int j = 0; j < 4; ++j) minv[4 * icol + j] *= pivinv;
        for (int j = 0; j < 4; ++j)
            if (j != icol) {
                const float save = minv[4 * j + icol];
                minv[4 * j + icol] = 0.0f;
                for (int k = 0; k < 4; ++k) minv[4 * j + k] -= minv[4 * icol + k] * save;
            }
    }
    for (int jj = 3; jj >= 0; --jj)
        if (indxr[jj] != indxc[jj])
            for (int k = 0; k < 4; ++k) { const float sw = minv[4 * k + indxr[jj]]; minv[4 * k + indxr[jj]] = minv[4 * k + indxc[jj]]; minv[4 * k + indxc[jj]] = sw; }
    for (int k = 0; k < 16; ++k) out[k] = minv[k];
}
PB_HD float quat_dot(const DQuat& a, const DQuat& b) { return a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w; }  // quaternion.rs:181-183

// ---- host: AnimatedTransform::new -------------------------------------------------------------------------------------------------
// AnimatedTransform::decompose (transform.rs:2032-2080)
inline void motion_decompose(const float* m, float* t, DQuat& q, float* s3) {
    t[0] = m[3]; t[1] = m[7]; t[2] = m[11];
    float r[16];
    for (int k = 0; k < 16; ++k) r[k] = m[k];
    for (int i = 0; i < 3; ++i) { r[4 * i + 3] = 0.0f; r[12 + i] = 0.0f; }
    r[15] = 1.0f;
    for (int count = 1;; ++count) {  // polar decomposition: R <- (R + R^-T) / 2
        float rt[16], rit[16], rnext[16];
        for (int i = 0; i < 4; ++i)
            for (int j = 0; j < 4; ++j) rt[4 * i + j] = r[4 * j + i];
        mx_inverse(rt, rit);
        for (int k = 0; k < 16; ++k) rnext[k] = 0.5f * (r[k] + rit[k]);
        float norm = 0.0f;
        for (int i = 0; i < 3; ++i) {
            const float n = fabsf(r[4 * i] - rnext[4 * i]) + fabsf(r[4 * i + 1] - rnext[4 * i + 1]) + fabsf(r[4 * i + 2] - rnext[4 * i + 2]);
            norm = fmaxf(norm, n);  // f32::max: a NaN operand yields the other
        }
        for (int k = 0; k < 16; ++k) r[k] = rnext[k];
        if (count >= 100 || norm <= 0.0001f) break;
    }
    // Quaternion::new (quaternion.rs:34-79)
    const float trace = r[0] + r[5] + r[10];
    if (trace > 0.0f) {
        float sq = sqrtf(trace + 1.0f);
        q.w = sq / 2.0f;
        sq = 0.5f / sq;
        q.x = (r[9] - r[6]) * sq; q.y = (r[2] - r[8]) * sq; q.z = (r[4] - r[1]) * sq;
    } else {
        const int nxt[3] = {1, 2, 0};
        float qv[3] = {0.0f, 0.0f, 0.0f};
        int i = r[5] > r[0] ? 1 : 0;
        if (r[10] > r[5 * i]) i = 2;
        const int j = nxt[i], k = nxt[j];
        float sq = sqrtf((r[5 * i] - (r[5 * j] + r[5 * k])) + 1.0f);
        qv[i] = sq * 0.5f;
        if (sq != 0.0f) sq = 0.5f / sq;
        q.w = (r[4 * k + j] - r[4 * j + k]) * sq;
        qv[j] = (r[4 * j + i] + r[4 * i + j]) * sq;
        qv[k] = (r[4 * k + i] + r[4 * i + k]) * sq;
        q.x = qv[0]; q.y = qv[1]; q.z = qv[2];
    }
    float rinv[16], sm[16];
    mx_inverse(r, rinv);
    mx_mul(rinv, m, sm);  // S = R^-1 M
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) s3[3 * i + j] = sm[4 * i + j];
}
// AnimatedTransform::new (transform.rs:912-932), without the derivative terms
inline void motion_create(const float* start, const float* start_inv, float start_time, const float* end, const float* end_inv, float end_time,
                          DMotion& mo) {
    for (int k = 0; k < 16; ++k) { mo.start[k] = start[k]; mo.start_inv[k] = start_inv[k]; mo.end[k] = end[k]; mo.end_inv[k] = end_inv[k]; }
    mo.start_time = start_time; mo.end_time = end_time;
    bool same = true;  // Transform's PartialEq: m and m_inv element-wise ==
    for (int k = 0; k < 16; ++k) same = same && start[k] == end[k] && start_inv[k] == end_inv[k];
    mo.actually_animated = same ? 0u : 1u;
    motion_decompose(start, mo.t[0], mo.r[0], mo.s[0]);
    motion_decompose(end, mo.t[1], mo.r[1], mo.s[1]);
    if (quat_dot(mo.r[0], mo.r[1]) < 0.0f) { mo.r[1].x = -mo.r[1].x; mo.r[1].y = -mo.r[1].y; mo.r[1].z = -mo.r[1].z; mo.r[1].w = -mo.r[1].w; }
    mo.has_rotation = quat_dot(mo.r[0], mo.r[1]) < 0.9995f ? 1u : 0u;
}

// ---- device: AnimatedTransform::interpolate (transform.rs:2081-2113) ---------------------------------------------------------------
// quat_normalize (quaternion.rs:186-188): q / |q|, where the vector part divides through Vector3f's `/`, a multiply by the
// reciprocal (geometry.rs:1271-1279), and w is divided
PB_HD DQuat quat_normalize(const DQuat& q) {
    const float l = sqrtf(quat_dot(q, q)), inv = 1.0f / l;
    DQuat o;
    o.x = q.x * inv; o.y = q.y * inv; o.z = q.z * inv; o.w = q.w / l;
    return o;
}
// quat_slerp (quaternion.rs:168-178)
PB_D DQuat quat_slerp(float t, const DQuat& q1, const DQuat& q2) {
    const float cos_theta = quat_dot(q1, q2);
    DQuat o;
    if (cos_theta > 0.9995f) {
        const float a = 1.0f - t;
        o.x = q1.x * a + q2.x * t; o.y = q1.y * a + q2.y * t; o.z = q1.z * a + q2.z * t; o.w = q1.w * a + q2.w * t;
        return quat_normalize(o);
    }
    const float theta = acos_rn(clampf(cos_theta, -1.0f, 1.0f));
    const float thetap = theta * t;
    DQuat qp;
    qp.x = q2.x - q1.x * cos_theta; qp.y = q2.y - q1.y * cos_theta; qp.z = q2.z - q1.z * cos_theta; qp.w = q2.w - q1.w * cos_theta;
    qp = quat_normalize(qp);
    float sn, cs;
    sincos_rn(thetap, sn, cs);
    o.x = q1.x * cs + qp.x * sn; o.y = q1.y * cs + qp.y * sn; o.z = q1.z * cs + qp.z * sn; o.w = q1.w * cs + qp.w * sn;
    return o;
}
// The transform at `time`: m and m_inv, composed as Transform's product composes them (transform.rs:869-877).  The boundary cases
// hand back the keyframes' own matrices.
PB_D void motion_interpolate(const DMotion& mo, float time, float* m, float* m_inv) {
    if (!mo.actually_animated || time <= mo.start_time) {
        for (int k = 0; k < 16; ++k) { m[k] = mo.start[k]; m_inv[k] = mo.start_inv[k]; }
        return;
    }
    if (time >= mo.end_time) {
        for (int k = 0; k < 16; ++k) { m[k] = mo.end[k]; m_inv[k] = mo.end_inv[k]; }
        return;
    }
    const float dt = (time - mo.start_time) / (mo.end_time - mo.start_time);
    const float tr[3] = {mo.t[0][0] * (1.0f - dt) + mo.t[1][0] * dt, mo.t[0][1] * (1.0f - dt) + mo.t[1][1] * dt, mo.t[0][2] * (1.0f - dt) + mo.t[1][2] * dt};
    const DQuat q = quat_slerp(dt, mo.r[0], mo.r[1]);
    float sc[16] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 1.0f};
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) sc[4 * i + j] = lerpf(dt, mo.s[0][3 * i + j], mo.s[1][3 * i + j]);
    float sc_inv[16];
    mx_inverse(sc, sc_inv);
    // Quaternion::to_transform (quaternion.rs:80-107): m = transpose(a), m_inv = a
    const float xx = q.x * q.x, yy = q.y * q.y, zz = q.z * q.z, xy = q.x * q.y, xz = q.x * q.z, yz = q.y * q.z, wx = q.x * q.w, wy = q.y * q.w,
                wz = q.z * q.w;
    const float a[16] = {1.0f - 2.0f * (yy + zz), 2.0f * (xy + wz), 2.0f * (xz - wy), 0.0f,
                         2.0f * (xy - wz), 1.0f - 2.0f * (xx + zz), 2.0f * (yz + wx), 0.0f,
                         2.0f * (xz + wy), 2.0f * (yz - wx), 1.0f - 2.0f * (xx + yy), 0.0f,
                         0.0f, 0.0f, 0.0f, 1.0f};
    float rot[16];
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) rot[4 * i + j] = a[4 * j + i];
    const float tm[16] = {1.0f, 0.0f, 0.0f, tr[0], 0.0f, 1.0f, 0.0f, tr[1], 0.0f, 0.0f, 1.0f, tr[2], 0.0f, 0.0f, 0.0f, 1.0f};
    const float tm_inv[16] = {1.0f, 0.0f, 0.0f, -tr[0], 0.0f, 1.0f, 0.0f, -tr[1], 0.0f, 0.0f, 1.0f, -tr[2], 0.0f, 0.0f, 0.0f, 1.0f};
    float tr_m[16], tr_inv[16];
    mx_mul(tm, rot, tr_m);         // (translate * rotate).m
    mx_mul(a, tm_inv, tr_inv);     // (translate * rotate).m_inv
    mx_mul(tr_m, sc, m);           // (.. * scale).m
    mx_mul(sc_inv, tr_inv, m_inv); // (.. * scale).m_inv
}

}  // namespace pb
