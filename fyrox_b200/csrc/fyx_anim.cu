// fyx_anim.cu — N2 (SURVEY §8f): the step right before the render-prep path, on the device.
//
// AnimationContainer::update_animations (scene/animation/mod.rs:83-88): every enabled animation ticks
// (Animation::tick, fyrox-animation/src/lib.rs:471-496: update_pose at the current time position, then the time
// advances) and its pose is applied to the nodes (AnimationPose::apply_internal / BoundValueCollection::apply,
// scene/animation/mod.rs:107-179).  Three launches per frame, nothing crosses PCIe:
//   k_anim_sample  one thread per track: Curve::value_at per component with the remembered span hints
//                  (fyrox-math/src/curve.rs:252-309), TrackDataContainer::fetch (fyrox-animation/src/container.rs:162-301)
//   k_anim_apply   one thread per animated node: its values in (animation, track) order through
//                  Transform::set_position / set_scale / set_rotation (scene/transform.rs:202-262: stored only if the
//                  transform is already dirty or the value differs), then Transform::calculate_local_transform
//   k_anim_tick    one thread per animation: set_time_position(time + dt * speed) (lib.rs:432-440: wrapf / clamp)
// Vector3 and UnitQuaternion tracks are bit-exact against the oracle; UnitQuaternionEuler tracks go through
// sin/cos, which the reference takes from the platform libm — those agree to ~1e-7, not bit for bit.
#include "fyx_internal.h"
#include "fyx_trs.cuh"

namespace fyx {

namespace {

__device__ __forceinline__ float sub_rn(const float a, const float b) { return FYX_ADD(a, -b); } // a - b == a + (-b) exactly

// fyrox-math/src/lib.rs:206-208
__device__ __forceinline__ float lerpf(const float a, const float b, const float t) { return FYX_ADD(a, FYX_MUL(sub_rn(b, a), t)); }

// fyrox-math/src/lib.rs:212-221 (sums left to right, products left to right)
__device__ __forceinline__ float cubicf(const float p0, const float p1, const float t, const float m0, const float m1)
{
    const float t2 = FYX_MUL(t, t);
    const float t3 = FYX_MUL(t2, t);
    const float scale = fabsf(sub_rn(p1, p0));
    const float a = FYX_MUL(FYX_ADD(sub_rn(FYX_MUL(2.0f, t3), FYX_MUL(3.0f, t2)), 1.0f), p0);
    const float b = FYX_MUL(FYX_MUL(FYX_ADD(sub_rn(t3, FYX_MUL(2.0f, t2)), t), m0), scale);
    const float c = FYX_MUL(FYX_ADD(FYX_MUL(-2.0f, t3), FYX_MUL(3.0f, t2)), p1);
    const float d = FYX_MUL(FYX_MUL(sub_rn(t3, t2), m1), scale);
    return FYX_ADD(FYX_ADD(FYX_ADD(a, b), c), d);
}

// CurveKey::interpolate (curve.rs:87-136): the left key's kind picks the family
__device__ __forceinline__ float key_interpolate(const fyx_curve_key &l, const fyx_curve_key &r, const float t)
{
    if (l.kind == FYX_KEY_CONSTANT) return (t == 1.0f) ? r.value : l.value; // stepf, curve.rs:25-31
    if (l.kind == FYX_KEY_LINEAR) return lerpf(l.value, r.value, t);
    return cubicf(l.value, r.value, t, l.right_tangent, (r.kind == FYX_KEY_CUBIC) ? r.left_tangent : 0.0f);
}

__device__ __forceinline__ float span_value(const fyx_curve_key &l, const fyx_curve_key &r, const float location)
{
    const float t = __fdiv_rn(sub_rn(location, l.location), sub_rn(r.location, l.location));
    return key_interpolate(l, r, t);
}

// Curve::value_at (curve.rs:252-309)
__device__ __forceinline__ float curve_value_at(const fyx_curve_key *keys, const uint32_t n, const float first_loc,
                                                const float last_loc, const float location, uint32_t &hint)
{
    if (n == 0u) return 0.0f;
    if (location <= first_loc) {
        hint = 0u;
        return keys[0].value;
    }
    if (location >= last_loc) {
        hint = n - 1u;
        return keys[n - 1u].value;
    }
    {
        const uint32_t h = hint, li = h ? h - 1u : 0u;
        if (li < n && h < n) {
            const fyx_curve_key pl = keys[li], pr = keys[h];
            if (location >= pl.location && location < pr.location) return span_value(pl, pr, location);
        }
    }
    uint32_t lo = 0u, hi = n; // partition_point(|k| k.location < location)
    while (lo < hi) {
        const uint32_t mid = lo + (hi - lo) / 2u;
        if (keys[mid].location < location) lo = mid + 1u;
        else hi = mid;
    }
    hint = lo;
    const uint32_t li = lo ? lo - 1u : 0u;
    if (lo >= n) return __int_as_float(0x7FC00000); // the reference would panic (NaN location): poison instead
    return span_value(keys[li], keys[lo], location);
}

// nalgebra: 4-component dot = (a0*b0 + a2*b2) + (a1*b1 + a3*b3); normalize = q_i / sqrt(dot(q, q))
__device__ __forceinline__ void quat_normalize(float q[4])
{
    const float n2 = FYX_ADD(FYX_ADD(FYX_MUL(q[0], q[0]), FYX_MUL(q[2], q[2])), FYX_ADD(FYX_MUL(q[1], q[1]), FYX_MUL(q[3], q[3])));
    const float n = __fsqrt_rn(n2);
    q[0] = __fdiv_rn(q[0], n);
    q[1] = __fdiv_rn(q[1], n);
    q[2] = __fdiv_rn(q[2], n);
    q[3] = __fdiv_rn(q[3], n);
}

// nalgebra quaternion product, components (i,j,k,w)
__device__ __forceinline__ void quat_mul(const float a[4], const float b[4], float o[4])
{
    const float w = sub_rn(sub_rn(sub_rn(FYX_MUL(a[3], b[3]), FYX_MUL(a[0], b[0])), FYX_MUL(a[1], b[1])), FYX_MUL(a[2], b[2]));
    const float i = sub_rn(FYX_ADD(FYX_ADD(FYX_MUL(a[3], b[0]), FYX_MUL(a[0], b[3])), FYX_MUL(a[1], b[2])), FYX_MUL(a[2], b[1]));
    const float j = FYX_ADD(FYX_ADD(sub_rn(FYX_MUL(a[3], b[1]), FYX_MUL(a[0], b[2])), FYX_MUL(a[1], b[3])), FYX_MUL(a[2], b[0]));
    const float k = FYX_ADD(sub_rn(FYX_ADD(FYX_MUL(a[3], b[2]), FYX_MUL(a[0], b[1])), FYX_MUL(a[1], b[0])), FYX_MUL(a[2], b[3]));
    o[0] = i; o[1] = j; o[2] = k; o[3] = w;
}

// quat_from_euler(v, RotationOrder::XYZ) = qz * qy * qx (fyrox-math/src/lib.rs:725-740)
__device__ __forceinline__ void quat_from_euler_xyz(const float e[3], float q[4])
{
    float s[3], c[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) sincosf(__fdiv_rn(e[a], 2.0f), &s[a], &c[a]);
    // from_axis_angle: (axis * sin, cos); the zero components are 0 * sin exactly as in the reference
    const float qx[4] = {FYX_MUL(1.0f, s[0]), FYX_MUL(0.0f, s[0]), FYX_MUL(0.0f, s[0]), c[0]};
    const float qy[4] = {FYX_MUL(0.0f, s[1]), FYX_MUL(1.0f, s[1]), FYX_MUL(0.0f, s[1]), c[1]};
    const float qz[4] = {FYX_MUL(0.0f, s[2]), FYX_MUL(0.0f, s[2]), FYX_MUL(1.0f, s[2]), c[2]};
    float t[4];
    quat_mul(qz, qy, t);
    quat_mul(t, qx, q);
}

__global__ void __launch_bounds__(kBlock) k_anim_sample(const AnimArrays an)
{
    const uint32_t i = blockIdx.x * kBlock + threadIdx.x;
    if (i >= an.n_tracks) return;
    const AnimTrackDev t = an.tracks[i];
    const AnimStateDev st = an.state[t.anim];
    if (!st.enabled) return; // nobody ticks a disabled animation: Animation::pose() keeps what the last tick left
    uint32_t ok = 0u;
    float4 out = make_float4(0.f, 0.f, 0.f, 0.f);
    const uint32_t need = (t.value_kind == FYX_TV_REAL) ? 1u : (t.value_kind == FYX_TV_VECTOR2) ? 2u
                          : (t.value_kind == FYX_TV_VECTOR3 || t.value_kind == FYX_TV_QUAT_EULER) ? 3u : 4u;
    if (t.enabled && t.n_curves >= need) {
        uint4 h4 = an.hints[i];
        uint32_t h[4] = {h4.x, h4.y, h4.z, h4.w};
        float v[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (uint32_t c = 0; c < 4u; ++c)
            if (c < need) v[c] = curve_value_at(an.keys + t.first_key[c], t.n_keys[c], t.first_loc[c], t.last_loc[c], st.time, h[c]);
        an.hints[i] = make_uint4(h[0], h[1], h[2], h[3]);
        if (t.value_kind == FYX_TV_QUAT_EULER) {
            float q[4];
            quat_from_euler_xyz(v, q);
            out = make_float4(q[0], q[1], q[2], q[3]);
        } else {
            if (t.value_kind == FYX_TV_QUAT) quat_normalize(v); // UnitQuaternion::from_quaternion
            out = make_float4(v[0], v[1], v[2], v[3]);
        }
        ok = 1u;
    }
    an.values[i] = out;
    an.value_ok[i] = ok;
}

// UnitQuaternion's PartialEq: equal coordinates or all negated
__device__ __forceinline__ bool quat_eq(const float a[4], const float4 b)
{
    if (a[0] == b.x && a[1] == b.y && a[2] == b.z && a[3] == b.w) return true;
    return a[0] == -b.x && a[1] == -b.y && a[2] == -b.z && a[3] == -b.w;
}

// Transform::set_position / set_scale / set_rotation through BoundValueCollection::apply (scene/animation/mod.rs:147-179)
struct ApplyState {
    fyx_trs t;
    bool dirty, touched;
};
__device__ __forceinline__ void apply_value(ApplyState &s, const uint32_t binding, const bool is_quat, const bool is_vec3, const float4 v)
{
    if (binding == FYX_BIND_POSITION && is_vec3) {
        s.touched = true;
        if (s.dirty || s.t.position[0] != v.x || s.t.position[1] != v.y || s.t.position[2] != v.z) {
            s.t.position[0] = v.x; s.t.position[1] = v.y; s.t.position[2] = v.z;
            s.dirty = true;
        }
    } else if (binding == FYX_BIND_SCALE && is_vec3) {
        s.touched = true;
        if (s.dirty || s.t.scale[0] != v.x || s.t.scale[1] != v.y || s.t.scale[2] != v.z) {
            s.t.scale[0] = v.x; s.t.scale[1] = v.y; s.t.scale[2] = v.z;
            s.dirty = true;
        }
    } else if (binding == FYX_BIND_ROTATION && is_quat) {
        s.touched = true;
        if (s.dirty || !quat_eq(s.t.rotation, v)) {
            s.t.rotation[0] = v.x; s.t.rotation[1] = v.y; s.t.rotation[2] = v.z; s.t.rotation[3] = v.w;
            s.dirty = true;
        }
    }
}

// TrackValue::blend_with (fyrox-animation/src/value.rs:201-227): nalgebra lerp a*(1-w) + b*w; rotations take the
// short way (value.rs:449-454) and are re-normalised
__device__ __forceinline__ float4 blend_value(const float4 a, const float4 b, const float w, const bool is_quat)
{
    const float u = sub_rn(1.0f, w);
    float s[4] = {a.x, a.y, a.z, a.w};
    if (is_quat) {
        const float d = FYX_ADD(FYX_ADD(FYX_MUL(s[0], b.x), FYX_MUL(s[2], b.z)), FYX_ADD(FYX_MUL(s[1], b.y), FYX_MUL(s[3], b.w)));
        if (d < 0.0f) { s[0] = -s[0]; s[1] = -s[1]; s[2] = -s[2]; s[3] = -s[3]; }
    }
    float o[4];
    o[0] = FYX_ADD(FYX_MUL(s[0], u), FYX_MUL(b.x, w));
    o[1] = FYX_ADD(FYX_MUL(s[1], u), FYX_MUL(b.y, w));
    o[2] = FYX_ADD(FYX_MUL(s[2], u), FYX_MUL(b.z, w));
    o[3] = is_quat ? FYX_ADD(FYX_MUL(s[3], u), FYX_MUL(b.w, w)) : 0.0f;
    if (is_quat) quat_normalize(o);
    return make_float4(o[0], o[1], o[2], o[3]);
}

// the output pose of a blend group for one node: at most one value per binding (duplicates are rejected when the group
// is made), kept in the order the first source pushed them
struct GroupPose {
    float4 v[3];
    uint32_t have, quat, order, n_order; // bit masks by binding; `order` packs the bindings 2 bits each
};
__device__ __forceinline__ void group_flush(GroupPose &gp, ApplyState &s)
{
    for (uint32_t k = 0; k < gp.n_order; ++k) {
        const uint32_t b = (gp.order >> (2u * k)) & 3u;
        const bool q = (gp.quat >> b) & 1u;
        apply_value(s, b, q, !q, gp.v[b]);
    }
    gp.have = gp.quat = gp.order = gp.n_order = 0u;
}

template <bool HAS_STATICS>
__global__ void __launch_bounds__(kBlock) k_anim_apply(const NodeArrays a, const AnimArrays an, fyx_trs *trs_by_slot,
                                                       const fyx_transform_statics *st_by_slot, uint32_t *d_err)
{
    const uint32_t e = blockIdx.x * kBlock + threadIdx.x;
    if (e >= an.n_nodes) return;
    const uint32_t slot = an.node_slot[e];
    ApplyState s;
    s.t = trs_by_slot[slot];
    s.dirty = s.touched = false; // Transform::dirty is clear after the last Graph::update
    GroupPose gp;
    gp.have = gp.quat = gp.order = gp.n_order = 0u;
    gp.v[0] = gp.v[1] = gp.v[2] = make_float4(0.f, 0.f, 0.f, 0.f);
    uint32_t cur_group = 0u, first_anim = FYX_NONE, cur_anim = FYX_NONE, src_done = 0u;
    // the node's tracks: direct animations first (animation, track order), then group after group, sources in group order
    for (uint32_t k = an.node_begin[e], k1 = an.node_begin[e + 1]; k < k1; ++k) {
        const uint32_t ti = an.node_tracks[k];
        const uint32_t anim = an.tracks[ti].anim;
        const AnimStateDev st = an.state[anim];
        if (st.group != cur_group) {
            if (cur_group) group_flush(gp, s);
            cur_group = st.group;
            first_anim = cur_anim = FYX_NONE;
        }
        if (!an.value_ok[ti]) continue;
        const float4 v = an.values[ti];
        const uint32_t bk = an.track_bind_kind[ti]; // binding | value_kind << 8
        const uint32_t binding = bk & 0xFFu, kind = bk >> 8;
        const bool is_quat = (kind == FYX_TV_QUAT || kind == FYX_TV_QUAT_EULER), is_vec3 = (kind == FYX_TV_VECTOR3);
        if (st.group == 0u) { // AnimationPlayer: only enabled animations tick and apply (scene/animation/mod.rs:84)
            if (st.enabled) apply_value(s, binding, is_quat, is_vec3, v);
            continue;
        }
        // blend group (BlendAnimations over PlayAnimation sources, machine/node/blend.rs:136-166, pose.rs:41-101)
        if (!(is_quat || is_vec3) || binding > FYX_BIND_ROTATION) continue;
        if (anim != cur_anim) { cur_anim = anim; src_done = 0u; }
        if (first_anim == FYX_NONE) first_anim = anim;
        const uint32_t bit = 1u << binding;
        if (anim == first_anim) { // the output has no values for this node yet: it takes a clone of the source's
            if (!(gp.have & bit)) {
                gp.order |= binding << (2u * gp.n_order);
                gp.n_order++;
            }
            gp.have |= bit;
            gp.quat = is_quat ? (gp.quat | bit) : (gp.quat & ~bit);
            gp.v[binding] = v;
        } else if ((gp.have & bit) && !(src_done & bit)) { // blended with the source's first value of that binding
            src_done |= bit;
            const bool oq = (gp.quat >> binding) & 1u;
            if (oq == is_quat) gp.v[binding] = blend_value(gp.v[binding], v, st.weight, oq);
        }
    }
    if (cur_group) group_flush(gp, s);
    if (!s.touched) return;
    if (s.dirty) trs_by_slot[slot] = s.t;
    Affine A;
    trs_to_local<HAS_STATICS>(s.t, HAS_STATICS ? st_by_slot + slot : nullptr, A);
    if (!(finite4(A.r0) & finite4(A.r1) & finite4(A.r2))) {
        atomicOr(d_err, E_NOT_AFFINE);
        return;
    }
    a.L[0][slot] = A.r0;
    a.L[1][slot] = A.r1;
    a.L[2][slot] = A.r2;
    atomicOr(a.flags + slot, F_DIRTY_SELF); // local_transform_mut(): NodeMessageKind::TransformChanged
}

// fyrox-math/src/lib.rs:179-203
__device__ __forceinline__ float wrapf(float n, float min_limit, float max_limit)
{
    if (n >= min_limit && n <= max_limit) return n;
    if (max_limit == 0.0f && min_limit == 0.0f) return 0.0f;
    max_limit = sub_rn(max_limit, min_limit);
    const float offset = min_limit;
    min_limit = 0.0f;
    n = sub_rn(n, offset);
    const float num_of_max = floorf(fabsf(__fdiv_rn(n, max_limit)));
    if (n >= max_limit) n = sub_rn(n, FYX_MUL(num_of_max, max_limit));
    else if (n < min_limit) n = FYX_ADD(n, FYX_MUL(FYX_ADD(num_of_max, 1.0f), max_limit));
    return FYX_ADD(n, offset);
}

__global__ void __launch_bounds__(kBlock) k_anim_tick(const AnimArrays an, const float dt)
{
    const uint32_t i = blockIdx.x * kBlock + threadIdx.x;
    if (i >= an.n_anims) return;
    AnimStateDev s = an.state[i];
    if (!s.enabled) return;
    const float nt = FYX_ADD(s.time, FYX_MUL(dt, s.speed));
    if (s.looped) {
        s.time = wrapf(nt, s.slice_start, s.slice_end);
    } else { // f32::clamp
        float x = nt;
        if (x < s.slice_start) x = s.slice_start;
        if (x > s.slice_end) x = s.slice_end;
        s.time = x;
    }
    an.state[i].time = s.time;
}

} // namespace

uint32_t launch_animate(cudaStream_t s, const NodeArrays &a, const AnimArrays &an, fyx_trs *trs_by_slot,
                        const fyx_transform_statics *st_by_slot, float dt, uint32_t *d_err)
{
    if (an.n_tracks) k_anim_sample<<<(an.n_tracks + kBlock - 1) / kBlock, kBlock, 0, s>>>(an);
    if (an.n_nodes) {
        const unsigned g = (an.n_nodes + kBlock - 1) / kBlock;
        if (st_by_slot) k_anim_apply<true><<<g, kBlock, 0, s>>>(a, an, trs_by_slot, st_by_slot, d_err);
        else k_anim_apply<false><<<g, kBlock, 0, s>>>(a, an, trs_by_slot, st_by_slot, d_err);
    }
    if (an.n_anims) k_anim_tick<<<(an.n_anims + kBlock - 1) / kBlock, kBlock, 0, s>>>(an, dt);
    return (an.n_tracks ? 1 : 0) + (an.n_nodes ? 1 : 0) + (an.n_anims ? 1 : 0);
}

} // namespace fyx
