// fyx_math.cuh — op-order-exact f32 arithmetic shared by the kernels.
//
// The reference is Rust + nalgebra: every `*` and `+` rounds once, nothing is contracted into FMA
// (SURVEY.md Appendix A).  On the device every product/sum therefore goes through __fmul_rn /
// __fadd_rn, which nvcc never fuses (the library is also built with -fmad=false).  Parenthesisation
// below IS the specification; do not "simplify".
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace fyx {

#if defined(__CUDA_ARCH__)
#define FYX_MUL(a, b) __fmul_rn((a), (b))
#define FYX_ADD(a, b) __fadd_rn((a), (b))
#else
#define FYX_MUL(a, b) ((a) * (b))
#define FYX_ADD(a, b) ((a) + (b))
#endif

// Affine 4x4 kept as its three upper rows; the bottom row is exactly (+0,+0,+0,1) for every matrix
// Transform::matrix() can produce (scene/transform.rs:476-539) and for every product of such
// matrices in nalgebra's order.  r[i] = (M[i,0], M[i,1], M[i,2], M[i,3]).
struct Affine {
    float4 r0, r1, r2;
};

__host__ __device__ __forceinline__ Affine affine_identity()
{
    Affine a;
    a.r0 = make_float4(1.f, 0.f, 0.f, 0.f);
    a.r1 = make_float4(0.f, 1.f, 0.f, 0.f);
    a.r2 = make_float4(0.f, 0.f, 1.f, 0.f);
    return a;
}

// One row of C = A·B for affine A, B in nalgebra's gemm order (Appendix A1):
//   C[i,j] = ((A[i,0]*B[0,j] + A[i,1]*B[1,j]) + A[i,2]*B[2,j]) + A[i,3]*B[3,j]
// with B[3,:] = (+0,+0,+0,1).  The A[i,3]*(+0) term is kept: it turns a -0 partial sum into +0
// exactly as the reference's full 4x4 product does.
__host__ __device__ __forceinline__ float4 affine_mul_row(const float4 a, const Affine &b)
{
    float4 c;
    const float z = FYX_MUL(a.w, 0.0f);
    c.x = FYX_ADD(FYX_ADD(FYX_ADD(FYX_MUL(a.x, b.r0.x), FYX_MUL(a.y, b.r1.x)), FYX_MUL(a.z, b.r2.x)), z);
    c.y = FYX_ADD(FYX_ADD(FYX_ADD(FYX_MUL(a.x, b.r0.y), FYX_MUL(a.y, b.r1.y)), FYX_MUL(a.z, b.r2.y)), z);
    c.z = FYX_ADD(FYX_ADD(FYX_ADD(FYX_MUL(a.x, b.r0.z), FYX_MUL(a.y, b.r1.z)), FYX_MUL(a.z, b.r2.z)), z);
    c.w = FYX_ADD(FYX_ADD(FYX_ADD(FYX_MUL(a.x, b.r0.w), FYX_MUL(a.y, b.r1.w)), FYX_MUL(a.z, b.r2.w)), a.w);
    return c;
}

// Graph::update_global_transform_recursively: G = parent.G * local (scene/graph/mod.rs:1216);
// palette: bone.G * inv_bind (scene/mesh/mod.rs:787-788).
__host__ __device__ __forceinline__ Affine affine_mul(const Affine &a, const Affine &b)
{
    Affine c;
    c.r0 = affine_mul_row(a.r0, b);
    c.r1 = affine_mul_row(a.r1, b);
    c.r2 = affine_mul_row(a.r2, b);
    return c;
}

// One row of AxisAlignedBoundingBox::transform (fyrox-math/src/aabb.rs:264-287, Appendix A4):
// min = max = M[i,3]; for j = 0,1,2: a = M[i,j]*lmin[j], b = M[i,j]*lmax[j]; a<b ? (min+=a,max+=b) : (min+=b,max+=a).
// Returns (min_i, max_i).
__host__ __device__ __forceinline__ float2 aabb_transform_row(const float4 row, const float2 lx, const float2 ly,
                                                              const float2 lz)
{
    float mn = row.w, mx = row.w;
    float a, b;
    a = FYX_MUL(row.x, lx.x); b = FYX_MUL(row.x, lx.y);
    if (a < b) { mn = FYX_ADD(mn, a); mx = FYX_ADD(mx, b); } else { mn = FYX_ADD(mn, b); mx = FYX_ADD(mx, a); }
    a = FYX_MUL(row.y, ly.x); b = FYX_MUL(row.y, ly.y);
    if (a < b) { mn = FYX_ADD(mn, a); mx = FYX_ADD(mx, b); } else { mn = FYX_ADD(mn, b); mx = FYX_ADD(mx, a); }
    a = FYX_MUL(row.z, lz.x); b = FYX_MUL(row.z, lz.y);
    if (a < b) { mn = FYX_ADD(mn, a); mx = FYX_ADD(mx, b); } else { mn = FYX_ADD(mn, b); mx = FYX_ADD(mx, a); }
    return make_float2(mn, mx);
}

// Pairwise f32 product / sum with ONE rounding per element.  sm_90 has no packed FP32 pipe, so each
// element is an ordinary __fmul_rn / __fadd_rn, which ptxas never contracts (the same results as the
// reference's separate `*` and `+`).  The `one` / `negzero` (1.0f, -0.0f) operands the packed FMA forms
// needed are no longer read; their plumbing through CullParams and the kernel parameters is left in place.
struct PackedConsts {
    float2 one, negzero;
};
__device__ __forceinline__ PackedConsts packed_consts(const float one = 1.0f, const float negzero = -0.0f)
{
    PackedConsts kc;
    kc.one = make_float2(one, one);
    kc.negzero = make_float2(negzero, negzero);
    return kc;
}
__device__ __forceinline__ float2 mul2(const float2 a, const float2 b, const PackedConsts &)
{
    return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y));
}
__device__ __forceinline__ float2 add2(const float2 a, const float2 c, const PackedConsts &)
{
    return make_float2(__fadd_rn(a.x, c.x), __fadd_rn(a.y, c.y));
}

// Frustum in kernel-parameter space.  planes as in frustum.rs:26-30; the 8 corners are kept as per-axis
// lists of distinct coordinates with the mask of corners sharing each (see the fallback below).
struct FrustumDev {
    float4 plane[6];
    float2 pn[3][4]; // planes (2q, 2q+1) as pairs: [q][0..2] = normal x,y,z pairs, [q][3] = d pair
    uint32_t cam_mask;
    uint32_t pass_flags;
    // vsel[q][axis][k]: byte-permute selector that picks, for plane 2q+k, the box bound whose product with the plane
    // normal's component on that axis is the larger one: 0x3210 = the minimum (component < 0), 0x7654 = the maximum.
    // One PRMT with a constant-bank operand per selected value (bit tests + predicate + SEL cost four).
    uint32_t vsel[3][3][2];
    uint32_t n_ax;   // n_ax >> (8*axis) & 0xFF: number of distinct corner coordinates on that axis
    // distinct corner coordinates per axis (unused entries are NaN: they compare false) and, for each, the
    // mask of the corners that have it
    float4 ax_val[3][2];
    uint32_t ax_mask[3][8]; // per distinct coordinate: the 8-bit mask of the frustum corners that have it
    // pm[q] = for planes (2q, 2q+1): the smallest s = ((nx*cx + ny*cy) + nz*cz) + d over the frustum's OWN eight corners,
    // evaluated on the host in exactly the kernels' arithmetic (NaN if any of them is NaN).  A box whose max-corner s on a
    // plane is below it cannot contain a frustum corner (see frustum_intersects_aabb): the fallback is skipped.
    float2 pm[3];
};

// Frustum::is_intersects_aabb (fyrox-math/src/frustum.rs:222-245) on (min,max) pairs per axis.
//
// Cloud test (frustum.rs:205-219): for each plane, all 8 corners have s = (n·p) + d <= 0  ⇒ outside.
// s(corner) = ((nx*px + ny*py) + nz*pz) + d with one rounding per op (plane.rs:78-80, Appendix A6).
// Rounding is monotone, so the corner built from the per-axis larger products has the largest s of
// the eight: "all eight <= 0"  ⇔  that corner's s <= 0 — the same booleans as the reference loop in
// 10 ops per plane instead of 56.  The argument needs NaN-free arithmetic and min <= max: boxes with a
// non-finite or huge (>1e18) bound or an inverted axis take the literal 8-corner loop instead (never in
// practice; the branch is uniform).
__device__ __forceinline__ bool aabb_is_tame(const float2 x, const float2 y, const float2 z)
{
    const float kBig = 1e18f;
    return (fabsf(x.x) <= kBig) & (fabsf(x.y) <= kBig) & (fabsf(y.x) <= kBig) & (fabsf(y.y) <= kBig) & (fabsf(z.x) <= kBig) &
           (fabsf(z.y) <= kBig) & (x.x <= x.y) & (y.x <= y.y) & (z.x <= z.y);
}

// prmt.b32 without __byte_perm's selector masking (the selectors are 0x3210 / 0x7654 by construction)
__device__ __forceinline__ float pick(const uint32_t lo, const uint32_t hi, const uint32_t sel)
{
    uint32_t d;
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(lo), "r"(hi), "r"(sel));
    return __uint_as_float(d);
}

__device__ __forceinline__ bool frustum_intersects_aabb(const FrustumDev &f, const float2 x, const float2 y,
                                                        const float2 z, const PackedConsts &kc, const bool tame)
{
    bool cloud = true, strong = false;
    if (tame) {
        // n*p is monotone in p (rounding is monotone), so max(fl(n*min), fl(n*max)) is fl(n*max) for n >= 0
        // and fl(n*min) for n < 0: pick the operand first (vsel, built on the host) and multiply once.
        // For n == ±0 both products are zeros; either choice gives the same booleans.
        // Two planes at a time: s = ((nx*vx + ny*vy) + nz*vz) + d element-wise.
        const uint32_t xl = __float_as_uint(x.x), xh = __float_as_uint(x.y), yl = __float_as_uint(y.x), yh = __float_as_uint(y.y),
                       zl = __float_as_uint(z.x), zh = __float_as_uint(z.y);
#pragma unroll
        for (int q = 0; q < 3; ++q) {
            const float2 vx = make_float2(pick(xl, xh, f.vsel[q][0][0]), pick(xl, xh, f.vsel[q][0][1]));
            const float2 vy = make_float2(pick(yl, yh, f.vsel[q][1][0]), pick(yl, yh, f.vsel[q][1][1]));
            const float2 vz = make_float2(pick(zl, zh, f.vsel[q][2][0]), pick(zl, zh, f.vsel[q][2][1]));
            const float2 s = add2(add2(add2(mul2(f.pn[q][0], vx, kc), mul2(f.pn[q][1], vy, kc), kc), mul2(f.pn[q][2], vz, kc), kc), f.pn[q][3], kc);
            cloud &= !(s.x <= 0.0f) & !(s.y <= 0.0f);
            strong |= (s.x < f.pm[q].x) | (s.y < f.pm[q].y);
            // siblings sit in adjacent slots, so a warp's boxes are usually cut off by the same plane: once every
            // lane here is rejected the remaining planes cannot change anything (a lane's own result never depends
            // on the vote: it only ever skips tests whose outcome is already fixed)
            if (q < 2 && !__any_sync(__activemask(), cloud)) break;
        }
    } else {
        // literal restatement of the 8-corner loop (NaN-correct).  Never taken in practice: kept rolled so that the
        // per-frustum code of the unrolled kernels stays small.
        const float xs[2] = {x.x, x.y}, ys[2] = {y.x, y.y}, zs[2] = {z.x, z.y};
#pragma unroll 1
        for (int p = 0; p < 6; ++p) {
            const float4 pl = f.plane[p];
            int back = 0;
#pragma unroll 1
            for (int c = 0; c < 8; ++c) {
                const float s = FYX_ADD(FYX_ADD(FYX_ADD(FYX_MUL(pl.x, (c & 1) ? xs[1] : xs[0]), FYX_MUL(pl.y, (c & 2) ? ys[1] : ys[0])),
                                                FYX_MUL(pl.z, (c & 4) ? zs[1] : zs[0])), pl.w);
                back += (s <= 0.0f) ? 1 : 0;
            }
            if (back >= 8) cloud = false;
        }
    }
    if (cloud) return true;
    // A frustum corner c inside the box (min <= c <= max on every axis) has, on every plane, s(c) <= s(max-corner of the box):
    // the per-axis products are monotone in the operand and the sums are monotone under round-to-nearest, in the very order
    // both are evaluated.  So a box whose max-corner s is BELOW the smallest s of the frustum's own corners on some plane
    // (pm, host-computed with the same operations) holds none of them: the fallback below would say false — skip it.
    // Only boxes that touch a plane within the rounding slack of the corners (|pm| ~ 1e-6 of the scene's size) go on.
    // CPU check of the claim: tests/test_cull_trick_cpu.py::test_strong_reject_skips_the_corner_fallback_exactly.
    if (strong) return false;
    // Fallback: any frustum corner inside the AABB, inclusive compares (aabb.rs:193-200):
    //   exists c: min <= corner_c <= max on all three axes.
    // Evaluated as three 8-bit corner masks (one per axis, built from the DISTINCT corner coordinates of
    // that axis — a frustum usually has <= 4) ANDed together, leaving after the first axis that no corner
    // satisfies: the same booleans as the reference's loop, ~15 instructions for the typical rejected box.
    uint32_t alive = 0xFFu;
    const float2 box[3] = {x, y, z};
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float lo = box[a].x, hi = box[a].y;
        const float4 v0 = f.ax_val[a][0];
        uint32_t m = 0u;
        m |= ((v0.x >= lo) & (v0.x <= hi)) ? f.ax_mask[a][0] : 0u;
        m |= ((v0.y >= lo) & (v0.y <= hi)) ? f.ax_mask[a][1] : 0u;
        m |= ((v0.z >= lo) & (v0.z <= hi)) ? f.ax_mask[a][2] : 0u;
        m |= ((v0.w >= lo) & (v0.w <= hi)) ? f.ax_mask[a][3] : 0u;
        if (((f.n_ax >> (8 * a)) & 0xFFu) > 4u) { // more than four distinct coordinates on this axis (uniform branch)
            const float4 v1 = f.ax_val[a][1];
            m |= ((v1.x >= lo) & (v1.x <= hi)) ? f.ax_mask[a][4] : 0u;
            m |= ((v1.y >= lo) & (v1.y <= hi)) ? f.ax_mask[a][5] : 0u;
            m |= ((v1.z >= lo) & (v1.z <= hi)) ? f.ax_mask[a][6] : 0u;
            m |= ((v1.w >= lo) & (v1.w <= hi)) ? f.ax_mask[a][7] : 0u;
        }
        alive &= m;
        if (!alive) return false;
    }
    return true;
}

} // namespace fyx
