"""Signals and root motion on the device (fyx_anim_set_signals / fyx_anim_set_root_motion) against the restatement in
root_motion_oracle.py: Animation::tick's signal check on the unwrapped time and update_root_motion (fyrox-animation/src/
lib.rs:471-661), and the blend machine's running root-motion blends (pose.rs:89-101, machine/mod.rs:344-385).  Root
motions, group root motions, drained events, lost counts, time positions and the global matrices and world boxes of
every node, bit for bit, every tick."""
import numpy as np
import pytest

import fyrox_b200 as fb
import oracle_binding as ob
import root_motion_oracle as rmo
from helpers import assert_same_hierarchy, bits_equal, camera_frustum
from test_gpu_anim import Builder, load_pair, make_graph

pytestmark = pytest.mark.gpu


def build_anim(rng, root, others, first_pos_elsewhere=False):
    """A root with a Position and a Rotation track, plus tracks on other nodes; optionally the animation's first
    Position track targets another node (the cycle-start / end values then come from it)."""
    b = Builder(rng)
    if first_pos_elsewhere:
        b.track(others[0], ob.BIND_POSITION, ob.TV_VECTOR3)
    b.track(root, ob.BIND_POSITION, ob.TV_VECTOR3, kinds=(1, 2))
    b.track(root, ob.BIND_ROTATION, ob.TV_QUAT, lo=-1.0, hi=1.0, kinds=(1, 2))
    for n in others:
        b.track(n, ob.BIND_ROTATION, ob.TV_QUAT, lo=-1.0, hi=1.0)
    return b.arrays()


def check_root_motions(ctx, anims, groups=()):
    got = ctx.anim_root_motions(0, len(anims))
    for i, a in enumerate(anims):
        dp, dr, present = rmo.root_motion_record(a.root_motion)
        assert got[i]["present"] == present, i
        assert bits_equal(got[i]["delta_position"], dp).all(), (i, got[i], dp)
        assert bits_equal(got[i]["delta_rotation"], dr).all(), (i, got[i], dr)
    if groups:
        got = ctx.anim_group_root_motions(1, len(groups))
        for g, grp in enumerate(groups):
            dp, dr, present = rmo.root_motion_record(grp.root_motion)
            assert got[g]["present"] == present, g
            assert bits_equal(got[g]["delta_position"], dp).all(), (g, got[g], dp)
            assert bits_equal(got[g]["delta_rotation"], dr).all(), (g, got[g], dr)


def check_events(ctx, anims, storage, first=None):
    """first: drain that many events first, then the rest (what does not fit stays queued, in order)."""
    ev, lost = ctx.anim_take_events(first)
    if first is not None:
        assert len(ev) <= first
        ev2, lost2 = ctx.anim_take_events()
        ev, lost = np.concatenate([ev, ev2]), lost + lost2
    want, want_lost = [], 0
    for i, a in enumerate(anims):
        e = a.take_events()
        want += [(i, s) for s in e[:storage[i]]]
        want_lost += max(0, len(e) - storage[i])
    assert [tuple(x) for x in ev.tolist()] == want
    assert lost == want_lost


def times_equal(ctx, anims):
    got = ctx.anim_time_positions(0, len(anims))
    assert bits_equal(got, np.array([a.time_position for a in anims], np.float32)).all()


@pytest.mark.parametrize("via_render_prep", [False, True])
def test_root_motion_and_signals_match_oracle(ctx, via_render_prep):
    rng = np.random.default_rng(2024 + via_render_prep)
    n = 400
    parent, flags, trs = make_graph(rng, n)
    og, tr = load_pair(ctx, parent, flags, trs)
    specs = [dict(speed=1.0, looped=True, time_slice=(0.0, 2.0), time_position=0.0),
             dict(speed=-1.5, looped=True, time_slice=(0.25, 2.0), time_position=1.0),
             dict(speed=2.5, looped=True, time_slice=(0.0, 1.5), time_position=0.5),
             dict(speed=0.0, looped=True, time_slice=(0.0, 2.0), time_position=0.75),
             dict(speed=1.0, looped=False, time_slice=(0.0, 2.0), time_position=0.0),
             dict(speed=0.75, looped=True, time_slice=(0.5, 2.25), time_position=0.5),
             dict(speed=1.25, looped=True, time_slice=(0.0, 2.0), time_position=0.0)]
    anims = []
    for i, kw in enumerate(specs):
        root = 10 + 40 * i
        t, k = build_anim(rng, root, list(range(root + 1, root + 12)), first_pos_elsewhere=(i == 5))
        anims.append(rmo.Animation(t, k, **kw))
        assert ctx.anim_add(t, k, **kw) == i
    settings = [dict(node=10), dict(node=50, ignore_y=True), dict(node=90, ignore_rotations=True), dict(node=130),
                None, dict(node=210, ignore_x=True, ignore_z=True), dict(node=250)]
    for i, s in enumerate(settings):
        if s is not None:
            anims[i].set_root_motion_settings(**s)
            ctx.anim_set_root_motion(i, **s)
    for i, a in enumerate(anims):
        sig = [(float(np.float32(rng.integers(0, 9) * 0.25)), bool(rng.random() < 0.85)) for _ in range(4)]
        for tm, en in sig:
            a.add_signal(tm, en)
        ctx.anim_set_signals(i, sig)
    # a small store: signals past it are dropped and counted (speed >= 0 only, so the queue length never differs)
    anims[6].max_event_capacity = 2
    ctx.anim_set_max_event_capacity(6, 2)
    storage = [max(a.max_event_capacity, len(a.signals)) for a in anims]
    _, ff = camera_frustum(zfar=500.0)
    dt = 0.125
    for frame in range(36):
        if frame == 6:
            anims[4].set_root_motion_settings(node=170)  # settings set mid-play: measured from prev_position 0
            ctx.anim_set_root_motion(4, node=170)
        if frame == 9:
            for a in (anims[1],):
                a.set_speed(0.5)
            ctx.anim_set_speed(1, 0.5)
            anims[2].set_time_position(1.375)
            ctx.anim_set_time_position(2, 1.375)
        if frame == 12:
            anims[3].set_enabled(False)
            ctx.anim_set_enabled(3, False)
            anims[0].signals[1][1] = not anims[0].signals[1][1]
            ctx.anim_set_signal_enabled(0, 1, anims[0].signals[1][1])
        if frame == 15:
            anims[0].set_root_motion_settings(None)  # the last root motion stays
            ctx.anim_set_root_motion(0)
            anims[6].set_track_enabled(1, False)  # the root's Position track: no value, default motion
            ctx.anim_set_track_enabled(6, 1, False)
        if frame == 18:
            anims[3].set_enabled(True)
            ctx.anim_set_enabled(3, True)
            anims[1].set_speed(-2.0)
            ctx.anim_set_speed(1, -2.0)
            anims[0].set_root_motion_settings(node=10, ignore_z=True)
            ctx.anim_set_root_motion(0, node=10, ignore_z=True)
        if frame == 22:
            dt = 0.3  # off the key grid
        rmo.update_animations(anims, dt, og, tr)
        og.update()
        if via_render_prep:
            ctx.render_prep(update_flags=fb.UPDATE_INCREMENTAL, frusta=[ff], do_palettes=False, do_skin=False, animate_dt=dt)
        else:
            ctx.animate(dt)
            ctx.update_transforms(fb.UPDATE_INCREMENTAL)
        times_equal(ctx, anims)
        check_root_motions(ctx, anims)
        if frame % 4 != 3:  # some frames leave the events queued
            check_events(ctx, anims, storage, first=3 if frame % 5 == 0 else None)
        assert_same_hierarchy(og, ctx)


def test_group_root_motion_running_blends(ctx):
    rng = np.random.default_rng(77)
    n = 300
    parent, flags, trs = make_graph(rng, n)
    og, tr = load_pair(ctx, parent, flags, trs)
    specs = [dict(speed=1.0, looped=True, time_slice=(0.0, 2.0), time_position=0.0),
             dict(speed=-1.0, looped=True, time_slice=(0.0, 1.75), time_position=0.5),
             dict(speed=0.5, looped=True, time_slice=(0.0, 2.0), time_position=1.0),   # no settings
             dict(speed=1.5, looped=True, time_slice=(0.25, 2.0), time_position=0.25),
             dict(speed=1.0, looped=True, time_slice=(0.0, 2.0), time_position=0.5)]
    anims = []
    for i, kw in enumerate(specs):
        root = 20 if i < 3 else 120
        t, k = build_anim(rng, root, list(range(root + 1 + 10 * i, root + 9 + 10 * i)))
        anims.append(rmo.Animation(t, k, **kw))
        ctx.anim_add(t, k, **kw)
    for i, node in [(0, 20), (1, 20), (3, 120), (4, 120)]:
        anims[i].set_root_motion_settings(node=node)
        ctx.anim_set_root_motion(i, node=node)
    w1, w2 = [1.0, 0.5, 2.0], [0.0, 1.0]
    groups = [rmo.BlendGroup(anims[0:3], w1), rmo.BlendGroup(anims[3:5], w2)]
    assert ctx.anim_blend_group([0, 1, 2], w1) == 1
    assert ctx.anim_blend_group([3, 4], w2) == 2
    dt = 0.125
    for frame in range(30):
        if frame == 5:
            anims[1].set_enabled(False)  # a disabled source hands on its stale root motion
            ctx.anim_set_enabled(1, False)
        if frame == 10:
            groups[0].weights = [np.float32(w) for w in (0.5, 0.0, 1.0)]
            ctx.anim_set_blend_weights(1, [0.5, 0.0, 1.0])
            groups[1].weights = [np.float32(w) for w in (2.0, 0.5)]
            ctx.anim_set_blend_weights(2, [2.0, 0.5])
        if frame == 14:
            anims[1].set_enabled(True)
            ctx.anim_set_enabled(1, True)
        if frame == 20:
            dt = 0.3
        for g in groups:
            g.update(dt, og, tr)
        og.update()
        ctx.animate(dt)
        ctx.update_transforms(fb.UPDATE_INCREMENTAL)
        times_equal(ctx, anims)
        check_root_motions(ctx, anims, groups)
        assert_same_hierarchy(og, ctx)


def test_launch_counts_and_refusals(ctx):
    rng = np.random.default_rng(5)
    parent, flags, trs = make_graph(rng, 50)
    load_pair(ctx, parent, flags, trs)
    t, k = build_anim(rng, 3, [4, 5])
    ctx.anim_add(t, k, time_slice=(0.0, 2.0))
    ctx.anim_add(t, k, time_slice=(0.0, 2.0))
    assert ctx.anim_blend_group([1], [1.0]) == 1

    def launches(fn):
        c0 = ctx.kernel_launch_count()
        fn()
        return ctx.kernel_launch_count() - c0

    base = launches(lambda: ctx.animate(0.1))
    assert base == 3  # k_anim_sample, k_anim_apply, k_anim_tick: no feature, no extra launch
    rm = ctx.anim_root_motions(0, 2)
    assert (rm["present"] == 0).all() and (rm["delta_rotation"][:, 3] == 1).all()
    assert ctx.anim_group_root_motions(1, 1)["present"][0] == 1  # evaluated once: Some(default fold)
    ctx.anim_set_signals(0, [(0.5, True)])
    assert launches(lambda: ctx.animate(0.1)) == base  # signals ride in k_anim_tick
    ctx.anim_set_root_motion(0, node=3)
    assert launches(lambda: ctx.animate(0.1)) == base + 2  # k_anim_root_motion + k_anim_group_root_motion
    # refusals leave the state as it was
    b = Builder(rng)
    b.track(7, ob.BIND_POSITION, ob.TV_VECTOR3)
    b.track(7, ob.BIND_POSITION, ob.TV_VECTOR3)
    t2, k2 = b.arrays()
    a2 = ctx.anim_add(t2, k2)
    with pytest.raises(fb.FyxError):
        ctx.anim_set_root_motion(a2, node=7)  # two Position tracks on the root
    ctx.anim_set_root_motion(a2, node=8)  # no track on the node: allowed, default motion
    for bad in (lambda: ctx.anim_set_root_motion(9, node=3), lambda: ctx.anim_set_signals(9, []),
                lambda: ctx.anim_set_signal_enabled(0, 1, True), lambda: ctx.anim_set_signal_enabled(9, 0, True),
                lambda: ctx.anim_set_max_event_capacity(9, 4), lambda: ctx.anim_root_motions(2, 2),
                lambda: ctx.anim_group_root_motions(0, 1), lambda: ctx.anim_group_root_motions(1, 2)):
        with pytest.raises(fb.FyxError):
            bad()
    with pytest.raises(fb.FyxError):
        ctx._chk(ctx._lib.fyx_anim_set_signals(ctx._h, 0, 2, None))
    ev, lost = ctx.anim_take_events()
    assert lost == 0


def test_host_mirror_hands_signals_and_settings_to_the_device(ctx):
    """fyrox_b200.animation: AnimationSignal / RootMotionSettings go up with AnimationContainer.upload; events come back
    with the signal's id and name, and root_motion() with the device's values."""
    from fyrox_b200 import animation as am
    parent, flags, trs = make_graph(np.random.default_rng(9), 8)
    load_pair(ctx, parent, flags, trs)
    a = am.Animation("walk")
    tr = am.Track.new_position()
    for c, v in enumerate((2.0, 0.0, 0.0)):
        tr.frames.curves[c].add_key(am.CurveKey(0.0, 0.0, am.CurveKeyKind.linear()))
        tr.frames.curves[c].add_key(am.CurveKey(2.0, v, am.CurveKeyKind.linear()))
    a.add_track_with_binding(am.TrackBinding(3), tr)
    a.set_time_slice(0.0, 2.0)
    a.add_signal(am.AnimationSignal(id=41, name="step", time=0.5))
    a.set_root_motion_settings(am.RootMotionSettings(node=3, ignore_y_movement=True))
    cont = am.AnimationContainer()
    cont.add(a)
    ids = cont.upload(ctx)
    for _ in range(3):
        ctx.animate(0.25)
    assert cont.fetch_events(ctx, ids) == 0
    assert a.pop_event() == am.AnimationEvent(41, "step") and a.pop_event() is None
    cont.fetch_root_motions(ctx, ids)
    assert a.root_motion() == am.RootMotion((0.25, 0.0, 0.0), (0.0, 0.0, 0.0, 1.0))


def test_async_frames_in_flight(ctx):
    """fyx_render_prep with do_animate, two asynchronous frames in flight: the getters and the drain reflect every frame
    enqueued so far."""
    rng = np.random.default_rng(31)
    n = 200
    parent, flags, trs = make_graph(rng, n)
    og, tr = load_pair(ctx, parent, flags, trs)
    anims = []
    for i, kw in enumerate([dict(speed=1.0, looped=True, time_slice=(0.0, 2.0), time_position=0.0),
                            dict(speed=-1.25, looped=True, time_slice=(0.0, 1.5), time_position=1.0)]):
        root = 10 + 60 * i
        t, k = build_anim(rng, root, list(range(root + 1, root + 10)))
        anims.append(rmo.Animation(t, k, **kw))
        ctx.anim_add(t, k, **kw)
        anims[i].set_root_motion_settings(node=root)
        ctx.anim_set_root_motion(i, node=root)
        for tm in (0.25, 0.5, 1.0, 1.25):
            anims[i].add_signal(tm)
        ctx.anim_set_signals(i, [(0.25, True), (0.5, True), (1.0, True), (1.25, True)])
    _, ff = camera_frustum(zfar=500.0)
    in_flight = 0
    for frame in range(24):
        dt = 0.125 if frame < 12 else 0.3
        rmo.update_animations(anims, dt, og, tr)
        og.update()
        ctx.render_prep(update_flags=fb.UPDATE_INCREMENTAL, frusta=[ff], do_palettes=False, do_skin=False, readback_visible=True,
                        async_=True, animate_dt=dt)
        in_flight += 1
        if frame % 3 != 2:  # the getters while this frame (and often the previous) is in flight
            times_equal(ctx, anims)
            check_root_motions(ctx, anims)
            check_events(ctx, anims, [32, 32])
        if in_flight == 2:
            ctx.frame_wait()
            in_flight -= 1
    while in_flight:
        ctx.frame_wait()
        in_flight -= 1
    times_equal(ctx, anims)
    check_root_motions(ctx, anims)
    check_events(ctx, anims, [32, 32])
    ctx.update_transforms(fb.UPDATE_INCREMENTAL)
    assert_same_hierarchy(og, ctx)


def test_c4_size_sampled(ctx):
    """One root-motion animation (root Position + Rotation, 4 signals) per unit of 50 000 units, 8 ticks; root motions and
    events of every animation against the oracle run on a sample of them, and their roots' global matrices."""
    rng = np.random.default_rng(12)
    units = 50_000
    n = 1 + units
    parent = np.zeros(n, np.uint32)
    parent[0] = ob.NONE
    flags = np.full(n, fb.NODE_DEFAULT | fb.NODE_RENDERABLE, np.uint32)
    trs = np.zeros((n, 10), np.float32)
    trs[:, 6] = 1.0
    trs[:, 7:10] = 1.0
    ctx.set_topology(parent, flags)
    ctx.set_local_trs(trs)
    ctx.update_transforms(fb.UPDATE_ALL)
    sample = set(rng.choice(units, 24, replace=False).tolist()) | {0, units - 1}
    oracles = {}
    sig = [(0.25, True), (0.75, True), (1.25, True), (1.75, False)]
    for u in range(units):
        b = Builder(rng)
        b.track(1 + u, ob.BIND_POSITION, ob.TV_VECTOR3, kinds=(1,), key_range=(1, 4))
        b.track(1 + u, ob.BIND_ROTATION, ob.TV_QUAT, lo=-1.0, hi=1.0, kinds=(1,), key_range=(1, 4))
        t, k = b.arrays()
        kw = dict(speed=float(rng.choice([1.0, -1.0, 2.0])), looped=True, time_slice=(0.0, 2.0), time_position=float(rng.integers(0, 8) * 0.25))
        ctx.anim_add(t, k, **kw)
        ctx.anim_set_root_motion(u, node=1 + u)
        ctx.anim_set_signals(u, sig)
        if u in sample:
            a = rmo.Animation(t, k, **kw)
            a.set_root_motion_settings(node=1 + u)
            for tm, en in sig:
                a.add_signal(tm, en)
            oracles[u] = a
    for frame in range(8):
        dt = 0.125 if frame % 2 else 0.3
        for u, a in oracles.items():
            a.tick(dt)
        ctx.animate(dt)
        got = ctx.anim_root_motions(0, units)
        assert (got["present"] == 1).all()
        ev, lost = ctx.anim_take_events()
        assert lost == 0
        for u, a in oracles.items():
            dp, dr, _ = rmo.root_motion_record(a.root_motion)
            assert bits_equal(got[u]["delta_position"], dp).all() and bits_equal(got[u]["delta_rotation"], dr).all(), u
            assert ev["signal"][ev["anim"] == u].tolist() == a.take_events(), u
        ctx.update_transforms(fb.UPDATE_INCREMENTAL)
        G = ctx.get_global_matrices(np.array([1 + u for u in oracles], np.uint32))
        for row, (u, a) in zip(G, oracles.items()):
            pos = [a.pose_val[i] for i in range(2) if a.pose_ok[i] and a.tracks[i]["binding"] == ob.BIND_POSITION]
            if pos:
                assert bits_equal(row[12:15], pos[0][:3]).all(), u  # the root stays at the slice start's position
