/*
 * fyrox_anim_oracle.c — CPU restatement of the step BEFORE the render-prep path (SURVEY §8f N2):
 * curve sampling -> track values -> animation pose -> node local transforms.
 *
 * TEST INFRASTRUCTURE ONLY (see fyrox_oracle.h).  Every function cites the reference file:line it follows
 * (paths under /root/reference).  Pinned against the reference's own unit tests of this code:
 * fyrox-math/src/curve.rs test_curve / test_curve_key, fyrox-math/src/lib.rs test_wrapf
 * (tests/test_oracle_kat.py K11-K14), and test_quat_from_euler (K15: quat_mul's order reproduces nalgebra's from_euler_angles
 * bit for bit).  Animation::tick, track fetch, pose application have no reference tests:
 * "parity unpinned", source-following.  nalgebra (absent from the tree, semver 0.35) supplies Vector::lerp,
 * Quaternion lerp / normalize / mul and the 4-component dot; their op orders are restated from its published
 * source and are this file's definition:
 *   dot4(a,b)        = (a0*b0 + a2*b2) + (a1*b1 + a3*b3)              (base/blas.rs, dotx, U4 special case)
 *   lerp(a,b,t)      = a*(1-t) + b*t per component                     (base/interpolation.rs)
 *   normalize(q)     = q_i / sqrt(dot4(q,q))                           (Normed::unscale_mut)
 *   q*r              = Quaternion::new(w, i, j, k) with
 *       w = w1*w2 - i1*i2 - j1*j2 - k1*k2     i = w1*i2 + i1*w2 + j1*k2 - k1*j2
 *       j = w1*j2 - i1*k2 + j1*w2 + k1*i2     k = w1*k2 + i1*j2 - j1*i2 + k1*w2   (geometry/quaternion_ops.rs)
 * sin/cos of the Euler path come from the platform libm exactly as Rust's f32::sin_cos does.
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "fyrox_oracle.h"

/* ---- fyrox-math/src/lib.rs ---- */

/* lib.rs:179-203 */
float orc_wrapf(float n, float min_limit, float max_limit)
{
    if (n >= min_limit && n <= max_limit) return n;
    if (max_limit == 0.0f && min_limit == 0.0f) return 0.0f;
    max_limit -= min_limit;
    float offset = min_limit;
    min_limit = 0.0f;
    n -= offset;
    float num_of_max = floorf(fabsf(n / max_limit));
    if (n >= max_limit) n -= num_of_max * max_limit;
    else if (n < min_limit) n += (num_of_max + 1.0f) * max_limit;
    return n + offset;
}

/* f32::clamp (core): NaN stays NaN; asserts min <= max */
static float clampf(float x, float lo, float hi)
{
    if (x < lo) x = lo;
    if (x > hi) x = hi;
    return x;
}

/* lib.rs:206-208 */
float orc_lerpf(float a, float b, float t) { return a + (b - a) * t; }

/* lib.rs:212-221 — Rust evaluates a + b + c + d left to right, x * y * z left to right */
float orc_cubicf(float p0, float p1, float t, float m0, float m1)
{
    float t2 = t * t;
    float t3 = t2 * t;
    float scale = fabsf(p1 - p0);
    float a = (2.0f * t3 - 3.0f * t2 + 1.0f) * p0;
    float b = (t3 - 2.0f * t2 + t) * m0 * scale;
    float c = (-2.0f * t3 + 3.0f * t2) * p1;
    float d = (t3 - t2) * m1 * scale;
    return a + b + c + d;
}

/* ---- fyrox-math/src/curve.rs ---- */

/* curve.rs:25-31 */
static float stepf(float p0, float p1, float t) { return (t == 1.0f) ? p1 : p0; }

/* curve.rs:87-136: the kind of the LEFT key selects the family, the right key only supplies its left tangent */
float orc_key_interpolate(const orc_curve_key *l, const orc_curve_key *r, float t)
{
    switch (l->kind) {
    case ORC_KEY_CONSTANT: return stepf(l->value, r->value, t);
    case ORC_KEY_LINEAR: return orc_lerpf(l->value, r->value, t);
    default:
        if (r->kind == ORC_KEY_CUBIC) return orc_cubicf(l->value, r->value, t, l->right_tangent, r->left_tangent);
        return orc_cubicf(l->value, r->value, t, l->right_tangent, 0.0f);
    }
}

/* Curve::fetch_at with the plain interpolator = Curve::value_at — curve.rs:252-309.  `hint` is the caller's
 * remembered span end (track.rs:31-34); the result depends on it when `location` sits exactly on a key. */
float orc_curve_value_at(const orc_curve_key *keys, uint32_t n, float location, uint32_t *hint)
{
    if (n == 0) return 0.0f;
    const orc_curve_key *first = &keys[0], *last = &keys[n - 1];
    if (location <= first->location) {
        *hint = 0;
        return first->value;
    }
    if (location >= last->location) {
        *hint = n - 1; /* len().saturating_sub(1) */
        return last->value;
    }
    /* NaN falls through both tests above, like the reference */
    {
        uint32_t h = *hint;
        uint32_t li = h ? h - 1 : 0; /* saturating_sub(1) */
        if (li < n && h < n) {
            const orc_curve_key *pl = &keys[li], *pr = &keys[h];
            if (location >= pl->location && location < pr->location) {
                float t = (location - pl->location) / (pr->location - pl->location);
                return orc_key_interpolate(pl, pr, t);
            }
        }
    }
    /* partition_point(|k| k.location < location): first index whose key is not < location (binary search) */
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
        uint32_t mid = lo + (hi - lo) / 2;
        if (keys[mid].location < location) lo = mid + 1;
        else hi = mid;
    }
    *hint = lo;
    {
        uint32_t li = lo ? lo - 1 : 0;
        if (li >= n || lo >= n) abort(); /* the reference unwraps; unreachable for non-NaN locations */
        const orc_curve_key *l = &keys[li], *r = &keys[lo];
        float t = (location - l->location) / (r->location - l->location);
        return orc_key_interpolate(l, r, t);
    }
}

/* ---- nalgebra pieces (see the header comment) ---- */
static float dot4(const float a[4], const float b[4]) { return (a[0] * b[0] + a[2] * b[2]) + (a[1] * b[1] + a[3] * b[3]); }

static void quat_normalize(float q[4])
{
    float n = sqrtf(dot4(q, q));
    q[0] = q[0] / n; q[1] = q[1] / n; q[2] = q[2] / n; q[3] = q[3] / n;
}

/* q = a * b, components (i,j,k,w) */
static void quat_mul(const float a[4], const float b[4], float out[4])
{
    float w = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
    float i = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1];
    float j = a[3] * b[1] - a[0] * b[2] + a[1] * b[3] + a[2] * b[0];
    float k = a[3] * b[2] + a[0] * b[1] - a[1] * b[0] + a[2] * b[3];
    out[0] = i; out[1] = j; out[2] = k; out[3] = w;
}

/* UnitQuaternion::from_axis_angle on a coordinate axis: (angle/2).sin_cos(), q = (axis*sin, cos) */
static void quat_axis_angle(int axis, float angle, float q[4])
{
    float h = angle / 2.0f;
    float s = sinf(h), c = cosf(h);
    q[0] = (axis == 0 ? 1.0f : 0.0f) * s;
    q[1] = (axis == 1 ? 1.0f : 0.0f) * s;
    q[2] = (axis == 2 ? 1.0f : 0.0f) * s;
    q[3] = c;
}

/* quat_from_euler(.., RotationOrder::XYZ) = qz * qy * qx — fyrox-math/src/lib.rs:725-740 */
void orc_quat_from_euler_xyz(const float e[3], float q[4])
{
    float qx[4], qy[4], qz[4], t[4];
    quat_axis_angle(0, e[0], qx);
    quat_axis_angle(1, e[1], qy);
    quat_axis_angle(2, e[2], qz);
    quat_mul(qz, qy, t);
    quat_mul(t, qx, q);
}

/* TrackValue::blend_with — fyrox-animation/src/value.rs:201-227: lerp for vectors, nlerp (shortest way) for rotations */
void orc_track_value_blend(int is_quat, float a[4], const float b[4], float w)
{
    if (!is_quat) {
        for (int i = 0; i < 4; ++i) a[i] = a[i] * (1.0f - w) + b[i] * w;
        return;
    }
    float s[4] = {a[0], a[1], a[2], a[3]};
    if (dot4(s, b) < 0.0f) { /* value.rs:449-454 */
        s[0] = -s[0]; s[1] = -s[1]; s[2] = -s[2]; s[3] = -s[3];
    }
    for (int i = 0; i < 4; ++i) a[i] = s[i] * (1.0f - w) + b[i] * w;
    quat_normalize(a);
}

/* TrackDataContainer::fetch — fyrox-animation/src/container.rs:162-301.  Returns 0 where the reference returns None. */
int orc_track_fetch(const orc_track *t, const orc_curve_key *keys, float time, uint32_t hints[4], float out[4])
{
    float v[4] = {0, 0, 0, 0};
    uint32_t need;
    switch (t->value_kind) {
    case ORC_TV_REAL: need = 1; break;
    case ORC_TV_VECTOR2: need = 2; break;
    case ORC_TV_VECTOR3: case ORC_TV_QUAT_EULER: need = 3; break;
    default: need = 4; break;
    }
    if (t->n_curves < need) return 0;
    for (uint32_t c = 0; c < need; ++c) v[c] = orc_curve_value_at(keys + t->first_key[c], t->n_keys[c], time, &hints[c]);
    if (t->value_kind == ORC_TV_QUAT_EULER) {
        orc_quat_from_euler_xyz(v, out);
    } else if (t->value_kind == ORC_TV_QUAT) {
        /* UnitQuaternion::from_quaternion(Quaternion::new(w, x, y, z)) = normalize */
        out[0] = v[0]; out[1] = v[1]; out[2] = v[2]; out[3] = v[3];
        quat_normalize(out);
    } else {
        memcpy(out, v, sizeof v);
    }
    return 1;
}

/* ---- Animation (fyrox-animation/src/lib.rs) ---- */
struct orc_animation {
    orc_track *tracks;
    uint32_t (*hints)[4]; /* TrackBinding::fetch_hints, track.rs:51 */
    uint32_t n_tracks;
    orc_curve_key *keys;
    uint32_t n_keys;
    float speed, time_position, slice_start, slice_end;
    int looped, enabled;
    /* Animation::pose (lib.rs:916-919): the values pushed by the last update_pose, in track order; it persists while the
     * animation is disabled (nobody ticks it), which a blend machine that still reads it can observe */
    float (*pose_val)[4];
    uint8_t *pose_ok;
};

orc_animation *orc_animation_new(const orc_track *tracks, uint32_t n_tracks, const orc_curve_key *keys, uint32_t n_keys)
{
    orc_animation *a = (orc_animation *)calloc(1, sizeof *a);
    a->tracks = (orc_track *)malloc(sizeof(orc_track) * (n_tracks ? n_tracks : 1));
    memcpy(a->tracks, tracks, sizeof(orc_track) * n_tracks);
    a->hints = (uint32_t(*)[4])calloc(n_tracks ? n_tracks : 1, sizeof(uint32_t[4]));
    a->pose_val = (float(*)[4])calloc(n_tracks ? n_tracks : 1, sizeof(float[4]));
    a->pose_ok = (uint8_t *)calloc(n_tracks ? n_tracks : 1, 1);
    a->n_tracks = n_tracks;
    a->keys = (orc_curve_key *)malloc(sizeof(orc_curve_key) * (n_keys ? n_keys : 1));
    memcpy(a->keys, keys, sizeof(orc_curve_key) * n_keys);
    a->n_keys = n_keys;
    /* Animation::default — lib.rs:922-945 */
    a->speed = 1.0f;
    a->time_position = 0.0f;
    a->enabled = 1;
    a->looped = 1;
    a->slice_start = a->slice_end = 0.0f;
    return a;
}

void orc_animation_free(orc_animation *a)
{
    if (!a) return;
    free(a->tracks);
    free(a->hints);
    free(a->pose_val);
    free(a->pose_ok);
    free(a->keys);
    free(a);
}

/* lib.rs:432-440 */
void orc_animation_set_time_position(orc_animation *a, float time)
{
    if (a->looped) a->time_position = orc_wrapf(time, a->slice_start, a->slice_end);
    else a->time_position = clampf(time, a->slice_start, a->slice_end);
}
/* lib.rs:445-452 */
void orc_animation_set_time_slice(orc_animation *a, float start, float end)
{
    a->slice_start = start;
    a->slice_end = end;
    orc_animation_set_time_position(a, a->time_position);
}
void orc_animation_set_speed(orc_animation *a, float s) { a->speed = s; }
void orc_animation_set_looped(orc_animation *a, int l) { a->looped = l; }
void orc_animation_set_enabled(orc_animation *a, int e) { a->enabled = e; }
void orc_animation_set_track_enabled(orc_animation *a, uint32_t t, int e) { if (t < a->n_tracks) a->tracks[t].enabled = (uint32_t)e; }
float orc_animation_time_position(const orc_animation *a) { return a->time_position; }
int orc_animation_is_enabled(const orc_animation *a) { return a->enabled; }

/* UnitQuaternion's PartialEq (nalgebra geometry/quaternion.rs): equal coordinates, or all negated (q and -q are the
 * same rotation) */
static int quat_eq(const float a[4], const float b[4])
{
    if (a[0] == b[0] && a[1] == b[1] && a[2] == b[2] && a[3] == b[3]) return 1;
    return a[0] == -b[0] && a[1] == -b[1] && a[2] == -b[2] && a[3] == -b[3];
}

/* Animation::tick (lib.rs:471-496): update_pose (lib.rs:895-914: pose.reset(), then per enabled track, in order,
 * fetch(time_position) and push into the target's NodePose), then the time position advances (signals / root
 * motion: out of scope). */
static void tick(orc_animation *a, float dt)
{
    for (uint32_t ti = 0; ti < a->n_tracks; ++ti) {
        const orc_track *t = &a->tracks[ti];
        a->pose_ok[ti] = 0;
        if (!t->enabled) continue;
        if (orc_track_fetch(t, a->keys, a->time_position, a->hints[ti], a->pose_val[ti])) a->pose_ok[ti] = 1;
    }
    orc_animation_set_time_position(a, a->time_position + dt * a->speed); /* lib.rs:474-491 */
}

/* One BoundValue reaching a node: BoundValueCollection::apply (scene/animation/mod.rs:147-179) through
 * Transform::set_position / set_scale / set_rotation (scene/transform.rs:202-262: stored only if the transform is
 * already dirty or the value differs), each via local_transform_mut() = TransformChanged.
 * dirty[n] = Transform::dirty of node n (cleared by the matrix() of the last Graph::update; see frame_dirty_or_new),
 * touched[n] = a TransformChanged message was sent. */
static void apply_value(uint32_t binding, int is_quat, int is_vec3, const float v[4], uint32_t n, const orc_graph *g,
                        orc_transform *transforms, uint32_t n_nodes, uint8_t *dirty, uint8_t *touched)
{
    if (n >= n_nodes || !orc_node_is_alive(g, n)) return; /* try_borrow_mut failed: logged and skipped */
    orc_transform *tr = &transforms[n];
    switch (binding) {
    case ORC_BIND_POSITION:
        if (!is_vec3) break; /* "underlying type is not Vector3": logged, skipped */
        touched[n] = 1;
        if (dirty[n] || tr->local_position[0] != v[0] || tr->local_position[1] != v[1] || tr->local_position[2] != v[2]) {
            memcpy(tr->local_position, v, 12);
            dirty[n] = 1;
        }
        break;
    case ORC_BIND_SCALE:
        if (!is_vec3) break;
        touched[n] = 1;
        if (dirty[n] || tr->local_scale[0] != v[0] || tr->local_scale[1] != v[1] || tr->local_scale[2] != v[2]) {
            memcpy(tr->local_scale, v, 12);
            dirty[n] = 1;
        }
        break;
    case ORC_BIND_ROTATION:
        if (!is_quat) break;
        touched[n] = 1;
        if (dirty[n] || !quat_eq(tr->local_rotation, v)) {
            memcpy(tr->local_rotation, v, 16);
            dirty[n] = 1;
        }
        break;
    default: break; /* ValueBinding::Property: reflection, out of scope */
    }
}

static int kind_is_quat(uint32_t k) { return k == ORC_TV_QUAT || k == ORC_TV_QUAT_EULER; }

/* AnimationPose::apply_internal of one animation's own pose.  Values of different nodes are independent, so walking
 * the tracks in order is the pose map walked in any order. */
static void apply_pose(const orc_animation *a, const orc_graph *g, orc_transform *transforms, uint32_t n_nodes,
                       uint8_t *dirty, uint8_t *touched)
{
    for (uint32_t ti = 0; ti < a->n_tracks; ++ti) {
        if (!a->pose_ok[ti]) continue;
        const orc_track *t = &a->tracks[ti];
        apply_value(t->binding, kind_is_quat(t->value_kind), t->value_kind == ORC_TV_VECTOR3, a->pose_val[ti], t->target_node, g,
                    transforms, n_nodes, dirty, touched);
    }
}

static void refresh_touched(orc_graph *g, orc_transform *transforms, uint32_t n_nodes, const uint8_t *touched)
{
    for (uint32_t k = 0; k < n_nodes; ++k)
        if (touched[k]) orc_node_set_local_transform(g, k, &transforms[k]);
}

/* Transform::dirty of every node for one frame.  Graph::update clears it (process_node_messages calls matrix() on
 * every transform that changed) and then updates the nodes in pool order (graph/mod.rs:1459-1504): the animation
 * players and the blend machines all apply their poses in that one loop and nothing calls matrix() between them, so
 * a transform a player set stays dirty for a machine that sets it later in the same frame.  `frame_dirty` is that
 * per-node flag, owned by the caller across the passes of one frame; NULL = a frame with this pass alone. */
static uint8_t *frame_dirty_or_new(uint8_t *frame_dirty, uint32_t n_nodes)
{
    return frame_dirty ? frame_dirty : (uint8_t *)calloc(n_nodes ? n_nodes : 1, 1);
}

/* AnimationContainer::update_animations — scene/animation/mod.rs:83-88: every enabled animation, in pool order,
 * ticks and applies its pose.  `transforms` = the nodes' Transform objects (indexed by node); the local matrices
 * of the touched nodes are then refreshed (what Transform::matrix() does lazily inside Graph::update) and a
 * TransformChanged message is queued for each. */
void orc_update_animations_in_frame(orc_animation **anims, uint32_t n, float dt, orc_graph *g, orc_transform *transforms,
                                    uint32_t n_nodes, uint8_t *frame_dirty)
{
    uint8_t *dirty = frame_dirty_or_new(frame_dirty, n_nodes);
    uint8_t *touched = (uint8_t *)calloc(n_nodes ? n_nodes : 1, 1);
    for (uint32_t i = 0; i < n; ++i)
        if (anims[i] && anims[i]->enabled) {
            tick(anims[i], dt);
            apply_pose(anims[i], g, transforms, n_nodes, dirty, touched);
        }
    refresh_touched(g, transforms, n_nodes, touched);
    if (dirty != frame_dirty) free(dirty);
    free(touched);
}

void orc_update_animations(orc_animation **anims, uint32_t n, float dt, orc_graph *g, orc_transform *transforms, uint32_t n_nodes)
{
    orc_update_animations_in_frame(anims, n, dt, g, transforms, n_nodes, NULL);
}

/* ---- blend machine, the smallest useful subset (fyrox-animation/src/machine) ----
 * One Machine with one layer, one state whose root is PoseNode::BlendAnimations over PoseNode::PlayAnimation sources
 * with constant weights, driving nodes through an AnimationPlayer with auto_apply = false:
 *   Machine::evaluate_pose (machine/mod.rs:344-382): every ENABLED animation the state uses ticks; the layer's pose is
 *   the state's pose (layer.rs:692-698, one state, no transition, no mask), final_pose = clone of it;
 *   BlendAnimations::eval_pose (machine/node/blend.rs:136-166): output.reset(); for each source in order
 *   output.blend_with(source pose, weight) where PlayAnimation::eval_pose (node/play.rs:86-100) is a clone of
 *   Animation::pose() — stale if that animation is disabled;
 *   AnimationPose::blend_with (pose.rs:87-101) / NodePose::blend_with (pose.rs:41-49) / BoundValueCollection::blend_with
 *   (value.rs:437-445): a node the output has no values for takes a CLONE of the source's values (the weight is not
 *   used), otherwise every output value is blended with the source's FIRST value of the same binding
 *   (TrackValue::blend_with, value.rs:201-227: same variant only);
 *   then the pose is applied (AnimationPoseExt::apply, scene/animation/mod.rs:117-125). */
typedef struct { uint32_t binding, is_quat, is_vec3; float v[4]; } pose_value;
typedef struct { pose_value *vals; uint32_t n, cap; } node_pose;

static void node_pose_push(node_pose *p, const pose_value *v)
{
    if (p->n == p->cap) {
        p->cap = p->cap ? p->cap * 2 : 4;
        p->vals = (pose_value *)realloc(p->vals, sizeof(pose_value) * p->cap);
    }
    p->vals[p->n++] = *v;
}

void orc_blend_group_update_in_frame(orc_animation **anims, const float *weights, uint32_t n, float dt, orc_graph *g,
                                     orc_transform *transforms, uint32_t n_nodes, uint8_t *frame_dirty)
{
    for (uint32_t i = 0; i < n; ++i) /* animations_cache is a set: an animation ticks once */
        if (anims[i] && anims[i]->enabled) {
            int seen = 0;
            for (uint32_t j = 0; j < i; ++j) seen |= (anims[j] == anims[i]);
            if (!seen) tick(anims[i], dt);
        }
    node_pose *out = (node_pose *)calloc(n_nodes ? n_nodes : 1, sizeof(node_pose));
    node_pose *src = (node_pose *)calloc(n_nodes ? n_nodes : 1, sizeof(node_pose));
    for (uint32_t s = 0; s < n; ++s) {
        const orc_animation *a = anims[s];
        if (!a) continue;
        /* the source's pose, grouped by node (values in track order) */
        for (uint32_t ti = 0; ti < a->n_tracks; ++ti) {
            if (!a->pose_ok[ti]) continue;
            const orc_track *t = &a->tracks[ti];
            if (t->target_node >= n_nodes) continue; /* would fail at apply; blending it changes nothing observable */
            pose_value pv;
            pv.binding = t->binding;
            pv.is_quat = (uint32_t)kind_is_quat(t->value_kind);
            pv.is_vec3 = (t->value_kind == ORC_TV_VECTOR3);
            memcpy(pv.v, a->pose_val[ti], 16);
            node_pose_push(&src[t->target_node], &pv);
        }
        for (uint32_t ti = 0; ti < a->n_tracks; ++ti) {
            if (!a->pose_ok[ti]) continue;
            const uint32_t nd = a->tracks[ti].target_node;
            if (nd >= n_nodes || !src[nd].n) continue; /* already merged (n reset below) */
            node_pose *o = &out[nd], *sp = &src[nd];
            if (o->n == 0) {
                for (uint32_t k = 0; k < sp->n; ++k) node_pose_push(o, &sp->vals[k]);
            } else {
                for (uint32_t k = 0; k < o->n; ++k) {
                    pose_value *ov = &o->vals[k];
                    for (uint32_t q = 0; q < sp->n; ++q)
                        if (sp->vals[q].binding == ov->binding) { /* find(): the first value with that binding */
                            if (ov->is_quat && sp->vals[q].is_quat) orc_track_value_blend(1, ov->v, sp->vals[q].v, weights[s]);
                            else if (ov->is_vec3 && sp->vals[q].is_vec3) {
                                float b4[4] = {sp->vals[q].v[0], sp->vals[q].v[1], sp->vals[q].v[2], 0.0f};
                                ov->v[3] = 0.0f;
                                orc_track_value_blend(0, ov->v, b4, weights[s]);
                            }
                            break;
                        }
                }
            }
            sp->n = 0;
        }
    }
    uint8_t *dirty = frame_dirty_or_new(frame_dirty, n_nodes);
    uint8_t *touched = (uint8_t *)calloc(n_nodes ? n_nodes : 1, 1);
    for (uint32_t nd = 0; nd < n_nodes; ++nd)
        for (uint32_t k = 0; k < out[nd].n; ++k) {
            const pose_value *pv = &out[nd].vals[k];
            apply_value(pv->binding, (int)pv->is_quat, (int)pv->is_vec3, pv->v, nd, g, transforms, n_nodes, dirty, touched);
        }
    refresh_touched(g, transforms, n_nodes, touched);
    for (uint32_t nd = 0; nd < n_nodes; ++nd) {
        free(out[nd].vals);
        free(src[nd].vals);
    }
    free(out);
    free(src);
    if (dirty != frame_dirty) free(dirty);
    free(touched);
}

void orc_blend_group_update(orc_animation **anims, const float *weights, uint32_t n, float dt, orc_graph *g,
                            orc_transform *transforms, uint32_t n_nodes)
{
    orc_blend_group_update_in_frame(anims, weights, n, dt, g, transforms, n_nodes, NULL);
}
