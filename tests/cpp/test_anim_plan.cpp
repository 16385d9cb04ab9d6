// N2's host rules (fyrox_b200/csrc/fyx_anim_plan.hpp) against the rules stated again here: the per-node track order of
// plan_anim_nodes on random animation sets over random forests (players and blend groups on one node, groups in any source
// order, dead / out-of-range / FYX_NONE targets, a topology change) and on the bench's shape; every refusal of fyx_anim_add
// and fyx_anim_blend_group just inside and just outside its limit; the device records of an added animation; time_position
// against the oracle's wrapf, bit for bit.  CPU only (built with -ffp-contract=off).  Prints "anim plan ok" when every check
// held.
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <random>
#include <string>
#include <vector>

#include "../../fyrox_b200/csrc/fyx_anim_plan.hpp"
#include "../../fyrox_b200/csrc/fyx_slots.hpp"
#include "../../fyrox_b200/csrc/scenegen.h"
#include "../../oracle/fyrox_oracle.h"

using namespace fyx;

static int g_fail = 0;
#define CHECK(cond, ...)                                                                            \
    do {                                                                                            \
        if (!(cond)) {                                                                              \
            if (g_fail++ < 20) {                                                                    \
                fprintf(stderr, "%s:%d: %s: ", __FILE__, __LINE__, #cond);                          \
                fprintf(stderr, __VA_ARGS__);                                                       \
                fprintf(stderr, "\n");                                                              \
            }                                                                                       \
        }                                                                                           \
    } while (0)

// The refusals of the checks: the message of the last one
static std::string g_msg;
static int32_t record(int32_t code, const char *fmt, ...)
{
    char buf[256];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_msg = buf;
    return code;
}

// ---- the per-node track order ----

// Animations as fyx_anim_add and fyx_anim_blend_group leave them: per animation its target nodes, and the blend groups
struct AnimSet {
    std::vector<std::vector<uint32_t>> targets; // per animation, per track
    std::vector<std::vector<uint32_t>> groups;  // sources of group g at [g - 1]
};

static void planner_inputs(const AnimSet &s, std::vector<AnimInfo> &anims, std::vector<uint32_t> &track_node)
{
    anims.clear();
    track_node.clear();
    for (const std::vector<uint32_t> &t : s.targets) {
        anims.push_back(AnimInfo{(uint32_t)track_node.size(), (uint32_t)t.size(), 1, 0.f, 1.f, 0, 0});
        track_node.insert(track_node.end(), t.begin(), t.end());
    }
    for (size_t g = 0; g < s.groups.size(); ++g)
        for (size_t i = 0; i < s.groups[g].size(); ++i) {
            anims[s.groups[g][i]].group = (uint32_t)g + 1;
            anims[s.groups[g][i]].pos_in_group = (uint32_t)i;
        }
}

// The order, stated without the planner's code: per live slot, the tracks of the directly applied animations in (animation,
// track) order, then for g = 1..G the tracks of group g's sources in the group's order
static AnimNodePlan expected(const AnimSet &s, const std::vector<uint32_t> &slot_of_node, uint32_t n_slots)
{
    std::vector<std::vector<uint32_t>> of_slot(n_slots);
    std::vector<uint32_t> first(s.targets.size());
    std::vector<bool> grouped(s.targets.size(), false);
    for (size_t a = 0, t = 0; a < s.targets.size(); t += s.targets[a].size(), ++a) first[a] = (uint32_t)t;
    for (const std::vector<uint32_t> &g : s.groups)
        for (uint32_t a : g) grouped[a] = true;
    auto add = [&](uint32_t a) {
        for (uint32_t k = 0; k < s.targets[a].size(); ++k) {
            const uint32_t node = s.targets[a][k];
            if (node < slot_of_node.size() && slot_of_node[node] != FYX_NONE) of_slot[slot_of_node[node]].push_back(first[a] + k);
        }
    };
    for (uint32_t a = 0; a < s.targets.size(); ++a)
        if (!grouped[a]) add(a);
    for (const std::vector<uint32_t> &g : s.groups)
        for (uint32_t a : g) add(a);
    AnimNodePlan p;
    for (uint32_t slot = 0; slot < n_slots; ++slot) {
        if (of_slot[slot].empty()) continue;
        p.node_slot.push_back(slot);
        p.node_begin.push_back((uint32_t)p.node_tracks.size());
        p.node_tracks.insert(p.node_tracks.end(), of_slot[slot].begin(), of_slot[slot].end());
    }
    p.node_begin.push_back((uint32_t)p.node_tracks.size());
    return p;
}

struct Forest {
    std::vector<uint32_t> parent, flags;
};

static void check_order(const AnimSet &s, const Forest &f, const char *what)
{
    const SlotPlan sp = plan_slots((uint32_t)f.parent.size(), f.parent.data(), f.flags.data());
    std::vector<AnimInfo> anims;
    std::vector<uint32_t> track_node;
    planner_inputs(s, anims, track_node);
    const AnimNodePlan got = plan_anim_nodes(anims, track_node, sp.slot_of_node);
    const AnimNodePlan want = expected(s, sp.slot_of_node, sp.n_slots());
    CHECK(got.node_slot == want.node_slot, "%s: node_slot differs (%zu vs %zu nodes)", what, got.node_slot.size(), want.node_slot.size());
    CHECK(got.node_begin == want.node_begin, "%s: node_begin differs", what);
    CHECK(got.node_tracks == want.node_tracks, "%s: node_tracks differs (%zu vs %zu tracks)", what, got.node_tracks.size(), want.node_tracks.size());
}

// parents earlier or out of range, some nodes dead
static Forest random_forest(std::mt19937_64 &rng, uint32_t n)
{
    Forest f;
    f.parent.resize(n);
    f.flags.assign(n, FYX_NODE_ALIVE);
    for (uint32_t i = 0; i < n; ++i) {
        f.parent[i] = (i == 0 || rng() % 10 == 0) ? FYX_NONE : (uint32_t)(rng() % i);
        if (rng() % 8 == 0) f.flags[i] = 0;
        if (rng() % 40 == 0) f.parent[i] = n + (uint32_t)(rng() % 3);
    }
    return f;
}

// random animations over n nodes: several tracks of one animation on one node, targets dead, out of range or FYX_NONE, and
// groups of random sources in random order (so a node is often driven by a player and by a group)
static AnimSet random_anims(std::mt19937_64 &rng, uint32_t n, uint32_t n_anims)
{
    AnimSet s;
    for (uint32_t a = 0; a < n_anims; ++a) {
        std::vector<uint32_t> t(rng() % 9);
        for (size_t k = 0; k < t.size(); ++k) {
            const uint32_t r = (uint32_t)(rng() % 20);
            if (r == 0) t[k] = FYX_NONE;
            else if (r == 1) t[k] = n + (uint32_t)(rng() % 5); // out of range
            else if (r < 5 && k) t[k] = t[k - 1];              // several tracks of one animation on one node
            else t[k] = n ? (uint32_t)(rng() % n) : 0;
        }
        s.targets.push_back(t);
    }
    std::vector<uint32_t> free_ids(n_anims);
    for (uint32_t a = 0; a < n_anims; ++a) free_ids[a] = a;
    std::shuffle(free_ids.begin(), free_ids.end(), rng);
    size_t at = 0;
    while (at < free_ids.size() && rng() % 3) {
        const size_t k = std::min<size_t>(1 + rng() % 4, free_ids.size() - at);
        s.groups.emplace_back(free_ids.begin() + at, free_ids.begin() + at + k); // source order is not id order
        at += k;
    }
    return s;
}

static void order_tests(std::mt19937_64 &rng)
{
    char what[160];
    check_order(AnimSet{}, Forest{}, "no nodes, no animations");
    {
        // node 1 by a player (animation 0, two tracks) and by group 1 (sources 3, 2); node 2 dead; 5 out of range
        const Forest f{{FYX_NONE, 0, 0, 1}, {FYX_NODE_ALIVE, FYX_NODE_ALIVE, 0, FYX_NODE_ALIVE}};
        AnimSet s;
        s.targets = {{1, 3, 1}, {2, 5, FYX_NONE}, {1, 3}, {3, 1}, {}};
        s.groups = {{3, 2}};
        check_order(s, f, "hand-made");
        const SlotPlan sp = plan_slots(4, f.parent.data(), f.flags.data());
        std::vector<AnimInfo> anims;
        std::vector<uint32_t> tn;
        planner_inputs(s, anims, tn);
        const AnimNodePlan p = plan_anim_nodes(anims, tn, sp.slot_of_node);
        // slots: 0 (node 0), 1 (node 1), 2 (node 3); node 1: tracks 0, 2 (animation 0), then 9 (animation 3), 6 (animation 2)
        CHECK(p.node_slot == std::vector<uint32_t>({1, 2}), "hand-made: animated slots");
        CHECK(p.node_begin == std::vector<uint32_t>({0, 4, 7}), "hand-made: node ranges");
        CHECK(p.node_tracks == std::vector<uint32_t>({0, 2, 9, 6, 1, 8, 7}), "hand-made: track order");
    }
    for (int t = 0; t < 600; ++t) {
        const uint32_t n = (uint32_t)(rng() % (t < 400 ? 40 : 3000));
        const Forest f = random_forest(rng, n);
        const AnimSet s = random_anims(rng, n, (uint32_t)(rng() % (t < 400 ? 12 : 400)));
        snprintf(what, sizeof what, "random set %d (%u nodes, %zu animations, %zu groups)", t, n, s.targets.size(), s.groups.size());
        check_order(s, f, what);
        // a topology change: nodes move (new parents) or die, the animations stay
        Forest g = f;
        for (uint32_t i = 0; i < n; ++i) {
            if (rng() % 6 == 0) g.flags[i] ^= FYX_NODE_ALIVE;
            if (i && rng() % 4 == 0) g.parent[i] = (uint32_t)(rng() % i);
        }
        snprintf(what, sizeof what, "random set %d after a topology change", t);
        check_order(s, g, what);
    }
}

// The bench's device animation: one animation per skinned unit, 64 rotation tracks on its bones with 4 keys per curve;
// checked with and without blend groups of units
static void bench_shape(uint32_t n_nodes, uint32_t n_units)
{
    const uint32_t bones = 64, K = 4;
    sg_config cfg{0xF1A0C5, n_nodes, n_units, bones, 100, 0, 1};
    sg_scene *sc = sg_create(&cfg);
    CHECK(sc, "scenegen refused %u nodes, %u units", n_nodes, n_units);
    if (!sc) return;
    Forest f{std::vector<uint32_t>(sg_parent(sc), sg_parent(sc) + sg_capacity(sc)), std::vector<uint32_t>(sg_flags(sc), sg_flags(sc) + sg_capacity(sc))};
    AnimSet s;
    std::vector<fyx_curve_key> keys(bones * 4 * K);
    for (uint32_t k = 0; k < keys.size(); ++k) keys[k] = fyx_curve_key{(float)(k % K) * (2.0f / 3.0f), 0.5f, FYX_KEY_LINEAR, 0.f, 0.f};
    std::vector<AnimTrackDev> recs;
    std::vector<uint32_t> bk;
    uint32_t n_keys = 0;
    for (uint32_t u = 0; u < sg_n_units(sc); ++u) {
        const uint32_t *b = sg_unit_bone_nodes(sc, u);
        s.targets.emplace_back(b, b + bones);
        std::vector<fyx_anim_track> tr(bones);
        for (uint32_t i = 0; i < bones; ++i) {
            tr[i] = fyx_anim_track{b[i], FYX_BIND_ROTATION, FYX_TV_QUAT, 1, 4, {}, {}};
            for (uint32_t c = 0; c < 4; ++c) tr[i].first_key[c] = (i * 4 + c) * K, tr[i].n_keys[c] = K;
        }
        const fyx_animation_desc d{sizeof(fyx_animation_desc), bones, tr.data(), (uint32_t)keys.size(), keys.data(), 1.f, 0.25f, 0.f, 2.f, 1, 1};
        CHECK(check_anim_desc(d, record) == FYX_OK, "bench shape: unit %u refused", u);
        append_anim(d, u, n_keys, recs, bk);
        n_keys += d.n_keys;
    }
    sg_free(sc);
    CHECK(recs.size() == (size_t)bones * s.targets.size() && recs.back().first_key[3] == n_keys - K, "bench shape: track records");
    check_order(s, f, "bench shape");
    for (uint32_t u = 0; u + 2 < s.targets.size(); u += 3) s.groups.push_back({u + 2, u}); // unit u + 1 stays a player
    check_order(s, f, "bench shape with blend groups");
}

// ---- fyx_anim_add ----

struct Desc {
    std::vector<fyx_anim_track> tracks;
    std::vector<fyx_curve_key> keys;
    fyx_animation_desc d;
    Desc(uint32_t n_keys = 6) : keys(n_keys)
    {
        for (uint32_t k = 0; k < n_keys; ++k) keys[k] = fyx_curve_key{0.5f * (float)k, (float)k, FYX_KEY_LINEAR, 0.f, 0.f};
        tracks.push_back(fyx_anim_track{0, FYX_BIND_POSITION, FYX_TV_VECTOR3, 1, 3, {0, 2, 4, 0}, {2, 2, 2, 0}});
        tracks.push_back(fyx_anim_track{0, FYX_BIND_ROTATION, FYX_TV_QUAT, 1, 4, {0, 1, 2, 3}, {3, 3, 3, 3}});
        d = fyx_animation_desc{sizeof(fyx_animation_desc), 0, nullptr, 0, nullptr, 1.f, 0.f, 0.f, 1.f, 1, 1};
    }
    const fyx_animation_desc &get()
    {
        d.n_tracks = (uint32_t)tracks.size();
        d.tracks = tracks.data();
        d.n_keys = (uint32_t)keys.size();
        d.keys = keys.data();
        return d;
    }
};

static void expect(int32_t rc, int32_t code, const char *msg, const char *what)
{
    CHECK(rc == code && g_msg == msg, "%s: got %d \"%s\", want %d \"%s\"", what, rc, g_msg.c_str(), code, msg);
    g_msg.clear();
}

static void add_refusals()
{
    const int32_t INV = FYX_ERR_INVALID_ARGUMENT, UNS = FYX_ERR_UNSUPPORTED;
    { Desc d; expect(check_anim_desc(d.get(), record), FYX_OK, "", "a valid description"); }
    // key range: the last key of a curve is the description's last key, or one past it (also where first + n wraps u32)
    { Desc d; d.tracks[1].first_key[2] = 3; expect(check_anim_desc(d.get(), record), FYX_OK, "", "curve ends on the last key"); }
    { Desc d; d.tracks[1].first_key[2] = 4; expect(check_anim_desc(d.get(), record), INV, "track 1 curve 2: keys out of range", "curve ends past the last key"); }
    { Desc d; d.tracks[0].first_key[1] = 0xFFFFFFFFu; expect(check_anim_desc(d.get(), record), INV, "track 0 curve 1: keys out of range", "first + n wraps"); }
    { Desc d; d.tracks[0].first_key[3] = 100; expect(check_anim_desc(d.get(), record), FYX_OK, "", "an unused curve's keys are not looked at"); }
    // curve count
    { Desc d; d.tracks[0].n_curves = 4; d.tracks[0].n_keys[3] = 1; expect(check_anim_desc(d.get(), record), FYX_OK, "", "4 curves"); }
    { Desc d; d.tracks[0].n_curves = 5; expect(check_anim_desc(d.get(), record), INV, "track 0: bad value kind / curve count", "5 curves"); }
    // value kind
    { Desc d; d.tracks[1].value_kind = FYX_TV_QUAT; expect(check_anim_desc(d.get(), record), FYX_OK, "", "last value kind"); }
    { Desc d; d.tracks[1].value_kind = FYX_TV_QUAT + 1; expect(check_anim_desc(d.get(), record), INV, "track 1: bad value kind / curve count", "value kind past the last"); }
    // binding
    { Desc d; d.tracks[0].binding = FYX_BIND_ROTATION; expect(check_anim_desc(d.get(), record), FYX_OK, "", "last binding"); }
    { Desc d; d.tracks[0].binding = FYX_BIND_ROTATION + 1; expect(check_anim_desc(d.get(), record), UNS, "track 0: property bindings are not supported", "property binding"); }
    // key kind
    { Desc d; d.keys[5].kind = FYX_KEY_CUBIC; expect(check_anim_desc(d.get(), record), FYX_OK, "", "cubic key"); }
    { Desc d; d.keys[5].kind = FYX_KEY_CUBIC + 1; expect(check_anim_desc(d.get(), record), INV, "key 5: bad kind", "key kind past cubic"); }
    // time slice: start <= end, NaN at either end refused
    const char *slice = "time slice start > end";
    { Desc d; d.d.time_slice_start = d.d.time_slice_end = 0.75f; expect(check_anim_desc(d.get(), record), FYX_OK, "", "zero-length slice"); }
    { Desc d; d.d.time_slice_start = nextafterf(1.f, 2.f); expect(check_anim_desc(d.get(), record), INV, slice, "start one ulp past end"); }
    { Desc d; d.d.time_slice_start = NAN; expect(check_anim_desc(d.get(), record), INV, slice, "NaN start"); }
    { Desc d; d.d.time_slice_end = NAN; expect(check_anim_desc(d.get(), record), INV, slice, "NaN end"); }
    // the slice is checked before the tracks, the tracks before the keys, each track's binding before its kind
    { Desc d; d.d.time_slice_end = -1.f; d.tracks[0].binding = 7; d.keys[0].kind = 9; expect(check_anim_desc(d.get(), record), INV, slice, "slice first"); }
    { Desc d; d.tracks[1].binding = 7; d.tracks[1].n_curves = 9; d.keys[0].kind = 9; expect(check_anim_desc(d.get(), record), UNS, "track 1: property bindings are not supported", "binding first"); }
    { Desc d; d.tracks.clear(); d.keys.clear(); expect(check_anim_desc(d.get(), record), FYX_OK, "", "no tracks, no keys"); }
}

static void track_records()
{
    Desc d;
    d.tracks[0].enabled = 7;
    d.tracks[0].target_node = 42;
    d.tracks[0].first_key[3] = 5; // an unused curve's fields are zeroed
    d.tracks[0].n_keys[3] = 1;
    d.tracks[1].n_keys[2] = 0; // an empty curve: no locations
    d.tracks[1].enabled = 0;
    d.d.speed = -2.5f;
    d.d.looped = 9;
    d.d.enabled = 0;
    d.d.time_slice_start = 0.25f;
    d.d.time_slice_end = 1.0f;
    d.d.time_position = 3.1f;
    std::vector<AnimTrackDev> recs(1, AnimTrackDev{});
    std::vector<uint32_t> bk(1, 99);
    const AnimStateDev st = append_anim(d.get(), 17, 1000, recs, bk);
    CHECK(recs.size() == 3 && bk.size() == 3, "records appended: %zu, %zu", recs.size(), bk.size());
    if (recs.size() != 3 || bk.size() != 3) return;
    const AnimTrackDev &a = recs[1], &b = recs[2];
    CHECK(bk[1] == (FYX_BIND_POSITION | FYX_TV_VECTOR3 << 8) && bk[2] == (FYX_BIND_ROTATION | FYX_TV_QUAT << 8), "binding | kind << 8");
    CHECK(a.anim == 17 && b.anim == 17 && a.value_kind == FYX_TV_VECTOR3 && a.enabled == 1 && b.enabled == 0 && a.n_curves == 3 && b.n_curves == 4,
          "track header");
    const uint32_t fk[4] = {1000, 1002, 1004, 0}, nk[4] = {2, 2, 2, 0};
    const float fl[4] = {0.f, 1.f, 2.f, 0.f}, ll[4] = {0.5f, 1.5f, 2.5f, 0.f};
    for (int k = 0; k < 4; ++k)
        CHECK(a.first_key[k] == fk[k] && a.n_keys[k] == nk[k] && a.first_loc[k] == fl[k] && a.last_loc[k] == ll[k], "track 0 curve %d", k);
    const uint32_t fk1[4] = {1000, 1001, 1002, 1003}, nk1[4] = {3, 3, 0, 3};
    const float fl1[4] = {0.f, 0.5f, 0.f, 1.5f}, ll1[4] = {1.f, 1.5f, 0.f, 2.5f};
    for (int k = 0; k < 4; ++k)
        CHECK(b.first_key[k] == fk1[k] && b.n_keys[k] == nk1[k] && b.first_loc[k] == fl1[k] && b.last_loc[k] == ll1[k], "track 1 curve %d", k);
    // the state: flags as 0 / 1, the time position wrapped into the slice
    CHECK(st.speed == -2.5f && st.slice_start == 0.25f && st.slice_end == 1.0f && st.looped == 1 && st.enabled == 0 && st.group == 0 &&
              st.weight == 0.f && st.time == orc_wrapf(3.1f, 0.25f, 1.0f),
          "state");
}

// ---- fyx_anim_blend_group ----

static void blend_refusals()
{
    const int32_t INV = FYX_ERR_INVALID_ARGUMENT, UNS = FYX_ERR_UNSUPPORTED;
    // animation 0: vector3 position + quat rotation on node 1; 1: quat-euler rotation on node 1 and node 2; 2: in group 1;
    // 3: a Real track; 4: two rotation tracks on node 2; 5: Vector2; 6: Vector4; 7: no tracks
    const std::vector<std::vector<std::pair<uint32_t, uint32_t>>> tr = {
        {{1, FYX_BIND_POSITION | FYX_TV_VECTOR3 << 8}, {1, FYX_BIND_ROTATION | FYX_TV_QUAT << 8}},
        {{1, FYX_BIND_ROTATION | FYX_TV_QUAT_EULER << 8}, {2, FYX_BIND_ROTATION | FYX_TV_QUAT << 8}},
        {{1, FYX_BIND_SCALE | FYX_TV_VECTOR3 << 8}},
        {{1, FYX_BIND_SCALE | FYX_TV_REAL << 8}},
        {{2, FYX_BIND_ROTATION | FYX_TV_QUAT << 8}, {3, FYX_BIND_SCALE | FYX_TV_VECTOR3 << 8}, {2, FYX_BIND_ROTATION | FYX_TV_QUAT_EULER << 8}},
        {{1, FYX_BIND_POSITION | FYX_TV_VECTOR2 << 8}},
        {{1, FYX_BIND_POSITION | FYX_TV_VECTOR4 << 8}},
        {}};
    std::vector<AnimInfo> anims;
    std::vector<uint32_t> node, bk;
    for (const auto &a : tr) {
        anims.push_back(AnimInfo{(uint32_t)node.size(), (uint32_t)a.size(), 0, 0.f, 1.f, 0, 0});
        for (const auto &t : a) node.push_back(t.first), bk.push_back(t.second);
    }
    anims[2].group = 1;
    const float w[4] = {0.5f, 0.25f, 1.f, 0.f};
    auto check = [&](std::vector<uint32_t> ids, int32_t code, const char *msg, const char *what) {
        expect(check_blend_group((uint32_t)ids.size(), ids.data(), w, anims, node, bk, record), code, msg, what);
    };
    check({0, 1}, FYX_OK, "", "vector3, quat and quat-euler sources");
    check({7}, FYX_OK, "", "a source without tracks");
    check({1, 0}, FYX_OK, "", "sources out of id order");
    const uint32_t one = 0;
    expect(check_blend_group(0, &one, w, anims, node, bk, record), INV, "empty blend group", "no sources");
    expect(check_blend_group(1, nullptr, w, anims, node, bk, record), INV, "empty blend group", "NULL sources");
    expect(check_blend_group(1, &one, nullptr, anims, node, bk, record), INV, "empty blend group", "NULL weights");
    check({0, 7}, FYX_OK, "", "the last animation");
    check({0, 8}, INV, "animation 8 does not exist", "one past the last animation");
    check({0, 2}, INV, "animation 2 already belongs to blend group 1", "a source already in a group");
    check({1, 0, 1}, INV, "animation 1 listed twice", "a source listed twice");
    check({3}, UNS, "animation 3 track 0: only Vector3 / UnitQuaternion tracks can be blended", "a Real track");
    check({5}, UNS, "animation 5 track 0: only Vector3 / UnitQuaternion tracks can be blended", "a Vector2 track");
    check({6}, UNS, "animation 6 track 0: only Vector3 / UnitQuaternion tracks can be blended", "a Vector4 track");
    check({0, 4}, UNS, "animation 4 animates one property of one node with two tracks", "two tracks on one (node, binding)");
    check({8, 3}, INV, "animation 8 does not exist", "sources checked in list order");
}

// ---- time_position ----

static bool same_bits(float a, float b) { return memcmp(&a, &b, 4) == 0; }

static void time_positions()
{
    // the slices and time classes of tests/anim_edges.py: inside, on the ends and one ulp either side, k lengths outside, far
    // outside (2^20 .. 2^24 lengths), negative; zero-length slices
    const float slices[][2] = {{0.1f, 0.7f}, {-1.f / 3.f, 5.f / 7.f}, {0.f, 2.f}, {0.f, 0.f}, {1.25f, 1.25f}, {1000.1f, 1003.7f}};
    int n = 0;
    for (const auto &sl : slices) {
        const float lo = sl[0], hi = sl[1], ln = hi - lo, base = std::max(ln, 1e-3f);
        std::vector<float> ts = {lo + ln * 0.5f, lo, hi, nextafterf(hi, -INFINITY), nextafterf(hi, INFINITY), nextafterf(lo, -INFINITY),
                                 nextafterf(lo, INFINITY), -0.3f, -7.9f, -1e3f, -std::fabs(lo) - 3.5f * ln - 1.f, 0.f, -0.f};
        for (float k : {2.f, 3.f, 7.f, -1.f, -2.f, -5.f}) ts.push_back(lo + k * ln);
        for (double q : {1048576.0, 8388608.0, 16777216.0})
            for (double sgn : {1.0, -1.0})
                for (double j : {-1.0, 0.0, 1.0}) ts.push_back((float)(lo + sgn * (q + j) * base + sgn * 0.37 * base));
        for (float t : ts) {
            AnimStateDev s{};
            s.slice_start = lo;
            s.slice_end = hi;
            s.looped = 1;
            const float got = time_position(s, t), want = orc_wrapf(t, lo, hi);
            CHECK(same_bits(got, want), "looped [%a, %a] at %a: %a, oracle %a", lo, hi, t, got, want);
            s.looped = 0; // f32::clamp
            const float clamped = time_position(s, t), cw = t < lo ? lo : (t > hi ? hi : t);
            CHECK(same_bits(clamped, cw), "clamped [%a, %a] at %a: %a, want %a", lo, hi, t, clamped, cw);
            const AnimInfo info{0, 0, 1, lo, hi, 0, 0};
            CHECK(same_bits(time_position(info, t), want), "an AnimInfo's time position at %a", t);
            ++n;
        }
    }
    CHECK(n > 200, "%d time positions", n);
}

int main()
{
    std::mt19937_64 rng(20261018);
    order_tests(rng);
    bench_shape(100000, 500);    // C4's 200 nodes per unit
    bench_shape(1000000, 10000); // C3
    add_refusals();
    track_records();
    blend_refusals();
    time_positions();
    if (g_fail) {
        fprintf(stderr, "%d checks failed\n", g_fail);
        return 1;
    }
    printf("anim plan ok\n");
    return 0;
}
