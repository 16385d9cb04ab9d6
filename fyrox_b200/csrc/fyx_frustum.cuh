// fyx_frustum.cuh — observer math shared by the host and the device: Frustum::from_view_projection_matrix, the kernels'
// frustum form (FrustumDev), and the look-at / perspective / product the shadow maps are built from.
//
// One implementation for both sides: the host builds the frusta fyx_cull receives, the device the frusta of
// fyx_cull_shadow_casters, and the two must agree bit for bit.  Every product / sum goes through FYX_MUL / FYX_ADD /
// FYX_SUB (never contracted: __fmul_rn & co. on the device, -ffp-contract=off on the host); ÷ and √ are IEEE on both
// (-prec-div, -prec-sqrt).
#pragma once
#include <math.h>
#include <string.h>

#include "../../include/fyrox_b200.h"
#include "fyx_math.cuh"

namespace fyx {

#if defined(__CUDA_ARCH__)
#define FYX_SUB(a, b) __fsub_rn((a), (b))
#else
#define FYX_SUB(a, b) ((a) - (b))
#endif

__host__ __device__ __forceinline__ uint32_t f32_bits(const float v)
{
    uint32_t u;
    memcpy(&u, &v, 4);
    return u;
}
__host__ __device__ __forceinline__ float f32_from_bits(const uint32_t u)
{
    float v;
    memcpy(&v, &u, 4);
    return v;
}
constexpr uint32_t kQuietNaN = 0x7FC00000u; // std::nanf("")
constexpr uint32_t kPlusInf = 0x7F800000u;

// nalgebra Vector3::dot, 3-element fast path: (a + b) + c (SURVEY Appendix A6)
__host__ __device__ __forceinline__ float dot3(const float *u, const float *v)
{
    return FYX_ADD(FYX_ADD(FYX_MUL(u[0], v[0]), FYX_MUL(u[1], v[1])), FYX_MUL(u[2], v[2]));
}
__host__ __device__ __forceinline__ void cross3(const float *u, const float *v, float *o)
{
    o[0] = FYX_SUB(FYX_MUL(u[1], v[2]), FYX_MUL(u[2], v[1]));
    o[1] = FYX_SUB(FYX_MUL(u[2], v[0]), FYX_MUL(u[0], v[2]));
    o[2] = FYX_SUB(FYX_MUL(u[0], v[1]), FYX_MUL(u[1], v[0]));
}

// Plane::from_abcd — fyrox-math/src/plane.rs:63-75
__host__ __device__ __forceinline__ bool plane_from_abcd(const float a, const float b, const float c, const float d, float *out)
{
    const float n[3] = {a, b, c};
    const float len = sqrtf(dot3(n, n));
    if (len == 0.0f) return false;
    const float coeff = 1.0f / len;
    out[0] = FYX_MUL(a, coeff);
    out[1] = FYX_MUL(b, coeff);
    out[2] = FYX_MUL(c, coeff);
    out[3] = FYX_MUL(d, coeff);
    return true;
}

// Plane::intersection_point — plane.rs:94-102
__host__ __device__ __forceinline__ void plane_intersection(const float *a, const float *b, const float *c, float *out)
{
    float bc[3], ca[3], ab[3];
    cross3(b, c, bc);
    const float f = -1.0f / dot3(a, bc);
    cross3(c, a, ca);
    cross3(a, b, ab);
    for (int i = 0; i < 3; ++i) out[i] = FYX_MUL(FYX_ADD(FYX_ADD(FYX_MUL(bc[i], a[3]), FYX_MUL(ca[i], b[3])), FYX_MUL(ab[i], c[3])), f);
}

// Frustum::from_view_projection_matrix — fyrox-math/src/frustum.rs:54-82; m[] is nalgebra's linear (column-major) index.
// false where the reference returns None (a zero-length plane normal).
__host__ __device__ __forceinline__ bool frustum_from_view_projection(const float *m, fyx_frustum &out)
{
    float(*p)[4] = out.planes;
    if (!plane_from_abcd(FYX_ADD(m[3], m[0]), FYX_ADD(m[7], m[4]), FYX_ADD(m[11], m[8]), FYX_ADD(m[15], m[12]), p[0])) return false;
    if (!plane_from_abcd(FYX_SUB(m[3], m[0]), FYX_SUB(m[7], m[4]), FYX_SUB(m[11], m[8]), FYX_SUB(m[15], m[12]), p[1])) return false;
    if (!plane_from_abcd(FYX_SUB(m[3], m[1]), FYX_SUB(m[7], m[5]), FYX_SUB(m[11], m[9]), FYX_SUB(m[15], m[13]), p[2])) return false;
    if (!plane_from_abcd(FYX_ADD(m[3], m[1]), FYX_ADD(m[7], m[5]), FYX_ADD(m[11], m[9]), FYX_ADD(m[15], m[13]), p[3])) return false;
    if (!plane_from_abcd(FYX_SUB(m[3], m[2]), FYX_SUB(m[7], m[6]), FYX_SUB(m[11], m[10]), FYX_SUB(m[15], m[14]), p[4])) return false;
    if (!plane_from_abcd(FYX_ADD(m[3], m[2]), FYX_ADD(m[7], m[6]), FYX_ADD(m[11], m[10]), FYX_ADD(m[15], m[14]), p[5])) return false;
    enum { L = 0, R = 1, T = 2, B = 3, F = 4, N = 5 }; // frustum.rs:70-79
    plane_intersection(p[L], p[T], p[F], out.corners[0]);
    plane_intersection(p[L], p[B], p[F], out.corners[1]);
    plane_intersection(p[R], p[B], p[F], out.corners[2]);
    plane_intersection(p[R], p[T], p[F], out.corners[3]);
    plane_intersection(p[L], p[T], p[N], out.corners[4]);
    plane_intersection(p[L], p[B], p[N], out.corners[5]);
    plane_intersection(p[R], p[B], p[N], out.corners[6]);
    plane_intersection(p[R], p[T], p[N], out.corners[7]);
    return true;
}

// Frustum → the kernels' form (FrustumDev, fyx_math.cuh)
__host__ __device__ __forceinline__ void to_dev_frustum(const fyx_frustum &f, const uint32_t cam_mask, const uint32_t pass_flags, FrustumDev &d)
{
    for (int p = 0; p < 6; ++p) d.plane[p] = make_float4(f.planes[p][0], f.planes[p][1], f.planes[p][2], f.planes[p][3]);
    for (int q = 0; q < 3; ++q)
        for (int k = 0; k < 4; ++k) d.pn[q][k] = make_float2(f.planes[2 * q][k], f.planes[2 * q + 1][k]);
    // distinct corner coordinates per axis (bit-pattern equality, so -0/+0 and NaNs stay separate entries:
    // each entry is compared exactly like the corner it came from)
    uint32_t n_ax = 0;
    for (int k = 0; k < 3; ++k) {
        int n = 0;
        uint32_t masks[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        float vals[8];
        for (int i = 0; i < 8; ++i) {
            const float v = f.corners[i][k];
            const uint32_t vb = f32_bits(v);
            int j = 0;
            for (; j < n; ++j)
                if (f32_bits(vals[j]) == vb) break;
            if (j == n) {
                vals[n] = v;
                ++n;
            }
            masks[j] |= 1u << i;
        }
        for (int j = n; j < 8; ++j) vals[j] = f32_from_bits(kQuietNaN); // never inside any box
        d.ax_val[k][0] = make_float4(vals[0], vals[1], vals[2], vals[3]);
        d.ax_val[k][1] = make_float4(vals[4], vals[5], vals[6], vals[7]);
        for (int j = 0; j < 8; ++j) d.ax_mask[k][j] = j < n ? masks[j] : 0u;
        n_ax |= (uint32_t)n << (8 * k);
    }
    d.n_ax = n_ax;
    d.cam_mask = cam_mask;
    d.pass_flags = pass_flags;
    for (int p = 0; p < 6; ++p)
        for (int k = 0; k < 3; ++k) d.vsel[p >> 1][k][p & 1] = (f.planes[p][k] < 0.0f) ? 0x3210u : 0x7654u;
    // smallest plane value over the frustum's own corners, one rounding per operation in the kernels' order
    for (int p = 0; p < 6; ++p) {
        float m = f32_from_bits(kPlusInf);
        for (int i = 0; i < 8; ++i) {
            const float v = FYX_ADD(FYX_ADD(FYX_ADD(FYX_MUL(f.planes[p][0], f.corners[i][0]), FYX_MUL(f.planes[p][1], f.corners[i][1])),
                                            FYX_MUL(f.planes[p][2], f.corners[i][2])),
                                    f.planes[p][3]);
            if (v != v || m != m) m = f32_from_bits(kQuietNaN);
            else if (v < m) m = v;
        }
        if (p & 1) d.pm[p >> 1].y = m;
        else d.pm[p >> 1].x = m;
    }
}

// Matrix4 * Matrix4 in nalgebra's accumulation order (Appendix A1): C[i,j] = ((A[i,0]B[0,j] + A[i,1]B[1,j]) + A[i,2]B[2,j]) + A[i,3]B[3,j]
__host__ __device__ __forceinline__ void mat4_mul(const float *a, const float *b, float *out)
{
    float r[16];
    for (int j = 0; j < 4; ++j)
        for (int i = 0; i < 4; ++i) {
            float y = FYX_MUL(a[i], b[j * 4]);
            y = FYX_ADD(y, FYX_MUL(a[4 + i], b[j * 4 + 1]));
            y = FYX_ADD(y, FYX_MUL(a[8 + i], b[j * 4 + 2]));
            y = FYX_ADD(y, FYX_MUL(a[12 + i], b[j * 4 + 3]));
            r[j * 4 + i] = y;
        }
    for (int k = 0; k < 16; ++k) out[k] = r[k];
}

// Matrix4::look_at_rh (nalgebra; the oracle's orc_look_at_rh), 16 f32 column-major
__host__ __device__ __forceinline__ void look_at_rh(const float *eye, const float *target, const float *up, float *out)
{
    float f[3] = {FYX_SUB(target[0], eye[0]), FYX_SUB(target[1], eye[1]), FYX_SUB(target[2], eye[2])};
    const float fl = sqrtf(dot3(f, f));
    f[0] = f[0] / fl;
    f[1] = f[1] / fl;
    f[2] = f[2] / fl;
    float s[3];
    cross3(f, up, s);
    const float sl = sqrtf(dot3(s, s));
    s[0] = s[0] / sl;
    s[1] = s[1] / sl;
    s[2] = s[2] / sl;
    float u[3];
    cross3(s, f, u);
    out[0] = s[0]; out[4] = s[1]; out[8] = s[2]; out[12] = -dot3(s, eye);
    out[1] = u[0]; out[5] = u[1]; out[9] = u[2]; out[13] = -dot3(u, eye);
    out[2] = -f[0]; out[6] = -f[1]; out[10] = -f[2]; out[14] = dot3(f, eye);
    out[3] = 0.0f; out[7] = 0.0f; out[11] = 0.0f; out[15] = 1.0f;
}

// Matrix4::new_perspective(aspect, fovy, znear, zfar) with m22 = 1 / tan(fovy / 2) given (nalgebra Perspective3::new)
__host__ __device__ __forceinline__ void perspective(const float m22, const float aspect, const float znear, const float zfar, float *out)
{
    for (int k = 0; k < 16; ++k) out[k] = 0.0f;
    out[5] = m22;
    out[0] = m22 / aspect;
    out[10] = FYX_ADD(zfar, znear) / FYX_SUB(znear, zfar);
    out[14] = FYX_MUL(FYX_MUL(zfar, znear), 2.0f) / FYX_SUB(znear, zfar);
    out[11] = -1.0f;
}

// The cascaded shadow maps' math (renderer/shadow/csm.rs:165-249).  nalgebra and approx have no source in the reference
// tree: look_at_lh, new_orthographic and relative_eq are restated from their documented definitions (unpinned), in the
// order of the oracle's orc_look_at_rh / orc_orthographic.

// Matrix4::new_orthographic(l, r, b, t, znear, zfar) (nalgebra Orthographic3::new; the oracle's orc_orthographic)
__host__ __device__ __forceinline__ void orthographic(const float l, const float r, const float b, const float t, const float zn, const float zf,
                                                      float *out)
{
    for (int k = 0; k < 16; ++k) out[k] = 0.0f;
    out[0] = 2.0f / FYX_SUB(r, l);
    out[5] = 2.0f / FYX_SUB(t, b);
    out[10] = -2.0f / FYX_SUB(zf, zn);
    out[12] = -FYX_ADD(r, l) / FYX_SUB(r, l);
    out[13] = -FYX_ADD(t, b) / FYX_SUB(t, b);
    out[14] = -FYX_ADD(zf, zn) / FYX_SUB(zf, zn);
    out[15] = 1.0f;
}

// Matrix4::look_at_lh (nalgebra: IsometryMatrix3::look_at_lh = Rotation3::face_towards(target − eye, up) inverted, then the
// rotation applied to −eye): rows s, u, f with f = normalize(target − eye), s = normalize(up × f), u = f × s
__host__ __device__ __forceinline__ void look_at_lh(const float *eye, const float *target, const float *up, float *out)
{
    float f[3] = {FYX_SUB(target[0], eye[0]), FYX_SUB(target[1], eye[1]), FYX_SUB(target[2], eye[2])};
    const float fl = sqrtf(dot3(f, f));
    f[0] = f[0] / fl;
    f[1] = f[1] / fl;
    f[2] = f[2] / fl;
    float s[3];
    cross3(up, f, s);
    const float sl = sqrtf(dot3(s, s));
    s[0] = s[0] / sl;
    s[1] = s[1] / sl;
    s[2] = s[2] / sl;
    float u[3];
    cross3(f, s, u);
    const float ne[3] = {-eye[0], -eye[1], -eye[2]};
    out[0] = s[0]; out[4] = s[1]; out[8] = s[2]; out[12] = dot3(s, ne);
    out[1] = u[0]; out[5] = u[1]; out[9] = u[2]; out[13] = dot3(u, ne);
    out[2] = f[0]; out[6] = f[1]; out[10] = f[2]; out[14] = dot3(f, ne);
    out[3] = 0.0f; out[7] = 0.0f; out[11] = 0.0f; out[15] = 1.0f;
}

// approx's relative_eq!(a, b) for f32 (epsilon = max_relative = f32::EPSILON)
__host__ __device__ __forceinline__ bool relative_eq(const float a, const float b)
{
    constexpr float eps = 1.1920929e-07f;
    if (a == b) return true;
    if (isinf(a) || isinf(b)) return false;
    const float d = fabsf(FYX_SUB(a, b));
    if (d <= eps) return true;
    const float aa = fabsf(a), ab = fabsf(b);
    const float largest = ab > aa ? ab : aa;
    return d <= FYX_MUL(largest, eps);
}

// Projection::with_z_near(zn).with_z_far(zf).matrix(frame_size) (scene/camera.rs:89-174).  Perspective: m22_or_vsize is
// 1 / tan(fov / 2) (evaluated on the host); orthographic: vertical_size.
__host__ __device__ __forceinline__ void camera_projection(const uint32_t kind, const float m22_or_vsize, const float z_near, const float z_far,
                                                           const float w, const float h, float *out)
{
    constexpr float limit = 1.1920929e-06f; // 10 * f32::EPSILON
    const float zn = fminf(z_far, z_near);
    float zf = fmaxf(z_far, z_near);
    if (FYX_SUB(zf, zn) < limit) zf = FYX_ADD(zf, limit);
    const float aspect = fmaxf(w / h, limit);
    if (kind == FYX_PROJECTION_PERSPECTIVE) {
        perspective(m22_or_vsize, aspect, zn, zf, out);
        return;
    }
    auto clamp_to_limit_signed = [](const float v) { return (v < 0.0f && -v < limit) ? -limit : (v >= 0.0f && v < limit) ? limit : v; };
    const float vs = clamp_to_limit_signed(m22_or_vsize);
    const float hs = clamp_to_limit_signed(FYX_MUL(aspect, vs));
    orthographic(-hs, hs, -vs, vs, zn, zf, out);
}

// Frustum::center (fyrox-math/src/frustum.rs:197-202): the corners folded from Vector3::default(), scaled by 1/8
__host__ __device__ __forceinline__ void frustum_center(const fyx_frustum &f, float *c)
{
    float a[3] = {0.0f, 0.0f, 0.0f};
    for (int i = 0; i < 8; ++i)
        for (int k = 0; k < 3; ++k) a[k] = FYX_ADD(a[k], f.corners[i][k]);
    for (int k = 0; k < 3; ++k) c[k] = FYX_MUL(a[k], 0.125f);
}

// Matrix4::transform_point (the oracle's orc_mat4_transform_point): (M3x3 p + t) / n, n = row3 · p + m33, unless n == 0
__host__ __device__ __forceinline__ void transform_point(const float *m, const float *p, float *out)
{
    const float n = FYX_ADD(FYX_ADD(FYX_ADD(FYX_MUL(m[3], p[0]), FYX_MUL(m[7], p[1])), FYX_MUL(m[11], p[2])), m[15]);
    float t[3];
    for (int i = 0; i < 3; ++i) t[i] = FYX_ADD(FYX_ADD(FYX_ADD(FYX_MUL(m[i], p[0]), FYX_MUL(m[4 + i], p[1])), FYX_MUL(m[8 + i], p[2])), m[12 + i]);
    if (n != 0.0f) {
        t[0] = t[0] / n;
        t[1] = t[1] / n;
        t[2] = t[2] / n;
    }
    out[0] = t[0]; out[1] = t[1]; out[2] = t[2];
}

} // namespace fyx
