// The signal and root-motion rules of fyx_anim_plan.hpp: the event rings of plan_events (offsets, storage =
// max(capacity, signals, queued), queued events kept in order, lost counts carried), the root-motion record of
// plan_root_motion (root tracks by kind, first Position / Rotation track of any target, ignore bits), check_root_motion's
// refusal at its limit, and plan_group_sources.  CPU only.  Prints
// "anim signal plan ok" when every check held.
#include <stdio.h>

#include <string>
#include <vector>

#include "../../fyrox_b200/csrc/fyx_anim_plan.hpp"

using namespace fyx;

static int g_fail = 0;
#define CHECK(cond)                                                           \
    do {                                                                      \
        if (!(cond) && g_fail++ < 20) fprintf(stderr, "%s:%d: %s\n", __FILE__, __LINE__, #cond); \
    } while (0)

static std::string g_msg;
static int32_t record(int32_t code, const char *fmt, ...)
{
    g_msg = fmt;
    return code;
}

static void rings()
{
    std::vector<AnimSignals> s(3);
    s[0].list = {{0.5f, 1u}, {1.0f, 0u}};
    s[1].cap = 2;
    s[1].list = {{0.1f, 1u}, {0.2f, 1u}, {0.3f, 1u}};
    s[2].cap = 1;
    const std::vector<std::vector<uint32_t>> queued = {{1, 0}, {}, {0, 0, 0}};
    const EventPlan p = plan_events(s, queued, {0u, 5u, 1u});
    CHECK(p.sig.size() == 3 && p.signals.size() == 5);
    CHECK(p.sig[0].ev_off == 0 && p.sig[0].storage == 32 && p.sig[0].count == 2 && p.sig[0].cap == 32);
    CHECK(p.sig[1].ev_off == 32 && p.sig[1].storage == 3 && p.sig[1].cap == 2 && p.sig[1].lost == 5); // the signals outnumber the capacity
    CHECK(p.sig[2].ev_off == 35 && p.sig[2].storage == 3 && p.sig[2].count == 3);                     // never below what is queued
    CHECK(p.sig[1].first_signal == 2 && p.sig[1].n_signals == 3 && p.sig[2].n_signals == 0);
    CHECK(p.events.size() == 38 && p.events[0] == 1 && p.events[1] == 0);
}

static void roots()
{
    // animation 0: tracks 0..5; node 4 has Position (Vector3) and Rotation (UnitQuaternionEuler); the first Position track
    // targets node 9, the first Rotation track node 4; a Vector4 Position track on node 5
    const std::vector<uint32_t> node = {9, 4, 4, 5, 4, 6};
    const std::vector<uint32_t> bk = {FYX_BIND_POSITION | FYX_TV_VECTOR3 << 8, FYX_BIND_ROTATION | FYX_TV_QUAT_EULER << 8,
                                      FYX_BIND_POSITION | FYX_TV_VECTOR3 << 8, FYX_BIND_POSITION | FYX_TV_VECTOR4 << 8,
                                      FYX_BIND_SCALE | FYX_TV_VECTOR3 << 8, FYX_BIND_ROTATION | FYX_TV_QUAT << 8};
    const AnimInfo a{0, 6, 1, 0.f, 1.f, 0, 0};
    fyx_root_motion_settings s{4, 1, 0, 1, 0};
    CHECK(check_root_motion(a, s, node, bk, record) == FYX_OK); // one Position, one Rotation, one Scale: allowed
    AnimRootDev r = plan_root_motion(3, a, s, node, bk);
    CHECK(r.anim == 3 && r.pos_track == 2 && r.rot_track == 1 && r.first_pos_track == 0 && r.first_rot_track == 1);
    CHECK(r.ignore == (kIgnoreX | kIgnoreZ));
    s.node = 5; // a Vector4 Position value never matches TrackValue::Vector3
    r = plan_root_motion(0, a, s, node, bk);
    CHECK(r.pos_track == FYX_NONE && r.rot_track == FYX_NONE);
    s.node = 77; // no track on the node: allowed
    CHECK(check_root_motion(a, s, node, bk, record) == FYX_OK);
    // just outside the limit: a second Position / Rotation track on the root
    std::vector<uint32_t> node2 = node, bk2 = bk;
    node2.push_back(4);
    bk2.push_back(FYX_BIND_POSITION | FYX_TV_VECTOR4 << 8);
    const AnimInfo a2{0, 7, 1, 0.f, 1.f, 0, 0};
    s.node = 4;
    CHECK(check_root_motion(a2, s, node2, bk2, record) == FYX_ERR_UNSUPPORTED);
    bk2.back() = FYX_BIND_ROTATION | FYX_TV_QUAT << 8;
    CHECK(check_root_motion(a2, s, node2, bk2, record) == FYX_ERR_UNSUPPORTED);
    bk2.back() = FYX_BIND_SCALE | FYX_TV_VECTOR3 << 8;
    CHECK(check_root_motion(a2, s, node2, bk2, record) == FYX_OK);
    // an animation's tracks only: a second Position track of the same node in ANOTHER animation does not count
    const AnimInfo a3{1, 6, 1, 0.f, 1.f, 0, 0};
    CHECK(check_root_motion(a3, s, node2, bk2, record) == FYX_OK);
}

static void group_sources()
{
    const GroupSourcePlan p = plan_group_sources({{4, 2}, {0}, {1, 3, 5}});
    CHECK((p.begin == std::vector<uint32_t>{0, 2, 3, 6}));
    CHECK((p.src == std::vector<uint32_t>{4, 2, 0, 1, 3, 5}));
}

int main()
{
    rings();
    roots();
    group_sources();
    if (g_fail) return 1;
    printf("anim signal plan ok\n");
    return 0;
}
