// fyx_anim_plan.hpp — N2's host rules: the checks of fyx_anim_add and fyx_anim_blend_group, the device records of an added
// animation, its time position on the host, and the per-node track order k_anim_apply blends in.  Host code only, with no
// CUDA types, so that the CPU tests build it with g++ alone.
#pragma once
#include <stdint.h>

#include <algorithm>
#include <cmath>
#include <vector>

#include "../../include/fyrox_b200.h"

namespace fyx {

// One track and one animation as k_anim_sample / k_anim_tick read them (fyx_anim.cu)
struct AnimTrackDev {
    uint32_t anim;       // owning animation
    uint32_t value_kind; // FYX_TV_*
    uint32_t enabled;
    uint32_t n_curves;
    uint32_t first_key[4]; // offsets into the context-wide key array
    uint32_t n_keys[4];
    float first_loc[4], last_loc[4]; // location of each curve's first / last key (keys are immutable once added): the
                                     // common in-range fetch touches only the remembered span, not the curve's ends
};
struct AnimStateDev {
    float time, speed, slice_start, slice_end;
    uint32_t looped, enabled;
    uint32_t group; // 0 = applied directly (AnimationPlayer, auto_apply); g > 0 = source of blend group g
    float weight;   // its PoseWeight::Constant inside that group
};

// What the host keeps of one animation
struct AnimInfo {
    uint32_t first_track, n_tracks; // its tracks in the context-wide track list
    uint32_t looped;
    float slice_start, slice_end;
    uint32_t group, pos_in_group; // its blend group (0 = applied directly) and its place among the group's sources
};

// fyrox-math/src/lib.rs:179-203 on the host (built with -ffp-contract=off)
inline float host_wrapf(float n, float min_limit, float max_limit)
{
    if (n >= min_limit && n <= max_limit) return n;
    if (max_limit == 0.0f && min_limit == 0.0f) return 0.0f;
    max_limit -= min_limit;
    const float offset = min_limit;
    min_limit = 0.0f;
    n -= offset;
    const float num_of_max = std::floor(std::fabs(n / max_limit));
    if (n >= max_limit) n -= num_of_max * max_limit;
    else if (n < min_limit) n += (num_of_max + 1.0f) * max_limit;
    return n + offset;
}

// Animation::set_time_position (fyrox-animation/src/lib.rs:432-440) of an AnimStateDev or an AnimInfo
template <class S> float time_position(const S &s, float t)
{
    if (s.looped) return host_wrapf(t, s.slice_start, s.slice_end);
    if (t < s.slice_start) t = s.slice_start;
    if (t > s.slice_end) t = s.slice_end;
    return t;
}

// The checks below refuse a call by returning fail(FYX_ERR_* code, printf format, arguments...); they return FYX_OK otherwise.

// fyx_anim_add's checks of a description whose arrays are present
template <class Fail> int32_t check_anim_desc(const fyx_animation_desc &d, Fail fail)
{
    if (!(d.time_slice_start <= d.time_slice_end)) return fail(FYX_ERR_INVALID_ARGUMENT, "time slice start > end"); // lib.rs:446 asserts
    for (uint32_t i = 0; i < d.n_tracks; ++i) {
        const fyx_anim_track &t = d.tracks[i];
        if (t.binding > FYX_BIND_ROTATION) return fail(FYX_ERR_UNSUPPORTED, "track %u: property bindings are not supported", i);
        if (t.value_kind > FYX_TV_QUAT || t.n_curves > 4) return fail(FYX_ERR_INVALID_ARGUMENT, "track %u: bad value kind / curve count", i);
        for (uint32_t k = 0; k < t.n_curves; ++k)
            if ((uint64_t)t.first_key[k] + t.n_keys[k] > d.n_keys) return fail(FYX_ERR_INVALID_ARGUMENT, "track %u curve %u: keys out of range", i, k);
    }
    for (uint32_t k = 0; k < d.n_keys; ++k)
        if (d.keys[k].kind > FYX_KEY_CUBIC) return fail(FYX_ERR_INVALID_ARGUMENT, "key %u: bad kind", k);
    return FYX_OK;
}

// The device records of a checked description: animation `id`'s tracks, whose keys start at k0 in the context-wide key array,
// onto `tracks` and their binding | value_kind << 8 onto `bind_kind`; the animation's state is the return value
inline AnimStateDev append_anim(const fyx_animation_desc &d, uint32_t id, uint32_t k0, std::vector<AnimTrackDev> &tracks,
                                std::vector<uint32_t> &bind_kind)
{
    for (uint32_t i = 0; i < d.n_tracks; ++i) {
        const fyx_anim_track &t = d.tracks[i];
        AnimTrackDev o{};
        o.anim = id;
        o.value_kind = t.value_kind;
        o.enabled = t.enabled ? 1u : 0u;
        o.n_curves = t.n_curves;
        for (int k = 0; k < 4; ++k) {
            o.first_key[k] = (k < (int)t.n_curves) ? k0 + t.first_key[k] : 0u;
            o.n_keys[k] = (k < (int)t.n_curves) ? t.n_keys[k] : 0u;
            if (o.n_keys[k]) {
                o.first_loc[k] = d.keys[t.first_key[k]].location;
                o.last_loc[k] = d.keys[t.first_key[k] + t.n_keys[k] - 1].location;
            }
        }
        tracks.push_back(o);
        bind_kind.push_back(t.binding | (t.value_kind << 8));
    }
    AnimStateDev st{};
    st.speed = d.speed;
    st.slice_start = d.time_slice_start;
    st.slice_end = d.time_slice_end;
    st.looped = d.looped ? 1u : 0u;
    st.enabled = d.enabled ? 1u : 0u;
    st.time = time_position(st, d.time_position);
    return st;
}

// fyx_anim_blend_group's checks of the sources ids[0..n) against the animations and their tracks (target node, binding |
// value_kind << 8 per track)
template <class Fail>
int32_t check_blend_group(uint32_t n, const uint32_t *ids, const float *weights, const std::vector<AnimInfo> &anims,
                          const std::vector<uint32_t> &track_node, const std::vector<uint32_t> &track_bind_kind, Fail fail)
{
    if (!n || !ids || !weights) return fail(FYX_ERR_INVALID_ARGUMENT, "empty blend group");
    std::vector<uint64_t> seen;
    for (uint32_t i = 0; i < n; ++i) {
        if (ids[i] >= anims.size()) return fail(FYX_ERR_INVALID_ARGUMENT, "animation %u does not exist", ids[i]);
        const AnimInfo &a = anims[ids[i]];
        if (a.group) return fail(FYX_ERR_INVALID_ARGUMENT, "animation %u already belongs to blend group %u", ids[i], a.group);
        for (uint32_t j = 0; j < i; ++j)
            if (ids[j] == ids[i]) return fail(FYX_ERR_INVALID_ARGUMENT, "animation %u listed twice", ids[i]);
        // inside a group every (node, property) has one track per animation, of a Vector3 / UnitQuaternion kind
        seen.clear();
        for (uint32_t t = 0; t < a.n_tracks; ++t) {
            const uint32_t bk = track_bind_kind[a.first_track + t], kind = bk >> 8;
            if (kind != FYX_TV_VECTOR3 && kind != FYX_TV_QUAT && kind != FYX_TV_QUAT_EULER)
                return fail(FYX_ERR_UNSUPPORTED, "animation %u track %u: only Vector3 / UnitQuaternion tracks can be blended", ids[i], t);
            seen.push_back(((uint64_t)track_node[a.first_track + t] << 2) | (bk & 0xFFu));
        }
        std::sort(seen.begin(), seen.end());
        if (std::adjacent_find(seen.begin(), seen.end()) != seen.end())
            return fail(FYX_ERR_UNSUPPORTED, "animation %u animates one property of one node with two tracks", ids[i]);
    }
    return FYX_OK;
}

// k_anim_apply's CSR: the animated nodes (distinct live targets, by slot) and, per node, its tracks
struct AnimNodePlan {
    std::vector<uint32_t> node_slot, node_begin, node_tracks; // node_begin: one entry per node, then the end
};

// Per node: the directly applied animations first (animation order), then blend group after blend group with the sources in
// the group's order; tracks in their own order inside an animation.  A target that is out of range or dead is skipped.
inline AnimNodePlan plan_anim_nodes(const std::vector<AnimInfo> &anims, const std::vector<uint32_t> &track_node,
                                    const std::vector<uint32_t> &slot_of_node)
{
    struct Ent { uint32_t slot, group, pos, track; };
    std::vector<Ent> st;
    st.reserve(track_node.size());
    for (uint32_t a = 0; a < anims.size(); ++a) {
        const AnimInfo &h = anims[a];
        for (uint32_t i = h.first_track; i < h.first_track + h.n_tracks; ++i) {
            const uint32_t node = track_node[i];
            if (node >= slot_of_node.size()) continue; // invalid handle: logged and skipped by the reference
            const uint32_t slot = slot_of_node[node];
            if (slot == FYX_NONE) continue;
            st.push_back(Ent{slot, h.group, h.group ? h.pos_in_group : a, i});
        }
    }
    std::stable_sort(st.begin(), st.end(), [](const Ent &x, const Ent &y) {
        if (x.slot != y.slot) return x.slot < y.slot;
        if (x.group != y.group) return x.group < y.group; // 0 = directly applied: first
        return x.pos < y.pos;                             // tracks of one animation keep their order (stable sort)
    });
    AnimNodePlan p;
    p.node_tracks.resize(st.size());
    for (size_t k = 0; k < st.size(); ++k) {
        if (k == 0 || st[k].slot != st[k - 1].slot) {
            p.node_slot.push_back(st[k].slot);
            p.node_begin.push_back((uint32_t)k);
        }
        p.node_tracks[k] = st[k].track;
    }
    p.node_begin.push_back((uint32_t)st.size());
    return p;
}

} // namespace fyx
