"""root_motion_oracle.py (signals, root motion and the blend machine's running root-motion blends) on hand-computed
dyadic cases, and, with neither feature set, against the C oracle's Animation::tick bit for bit.  CPU only."""
import ctypes as C

import numpy as np

import oracle_binding as ob
import root_motion_oracle as rmo

f32 = np.float32


def keys_tracks(spec):
    """spec: [(node, binding, kind, [curve keys [(loc, value, kind)]...])] -> (tracks, keys)"""
    keys, tracks = [], []
    for node, binding, kind, curves in spec:
        t = np.zeros((), ob.TRACK_DTYPE)
        t["target_node"], t["binding"], t["value_kind"], t["enabled"], t["n_curves"] = node, binding, kind, 1, len(curves)
        for c, curve in enumerate(curves):
            t["first_key"][c], t["n_keys"][c] = len(keys), len(curve)
            keys += [(loc, v, kd, 0.0, 0.0) for loc, v, kd in curve]
        tracks.append(t)
    k = np.zeros(len(keys), ob.KEY_DTYPE)
    for i, r in enumerate(keys):
        k[i] = r
    return np.array(tracks, ob.TRACK_DTYPE), k


LIN, CONST = ob.KEY_LINEAR, ob.KEY_CONSTANT
RAMP_X = [[(0.0, 0.0, LIN), (2.0, 2.0, LIN)], [(0.0, 3.0, CONST)], [(0.0, 0.0, CONST)]]  # x = t, y = 3, z = 0


def walk(speed=1.0, time_position=0.0, extra=()):
    t, k = keys_tracks([(1, ob.BIND_POSITION, ob.TV_VECTOR3, RAMP_X), *extra])
    return rmo.Animation(t, k, speed=speed, looped=True, time_slice=(0.0, 2.0), time_position=time_position)


def deltas(a, dt, n):
    out = []
    for _ in range(n):
        a.tick(dt)
        out.append(tuple(float(x) for x in a.root_motion.delta_position))
    return out


def test_loop_wrap_forward_keeps_velocity_through_the_remainder():
    a = walk()
    a.set_root_motion_settings(node=1)
    # poses at 0, 0.75, 1.5, then 0.25 after the wrap: the remainder fetch(2) - 1.5 = 0.5 carries the motion
    assert deltas(a, 0.75, 5) == [(0.0, 3.0, 0.0), (0.75, 0.0, 0.0), (0.75, 0.0, 0.0), (0.75, 0.0, 0.0), (0.75, 0.0, 0.0)]
    assert tuple(a.pose_val[0][:3]) == (0.0, 3.0, 0.0)  # reset to the slice start: the root stays in place
    assert a.root_motion.position_offset_remainder is None


def test_loop_wrap_backward():
    a = walk(speed=-1.0, time_position=2.0)
    a.set_root_motion_settings(node=1)
    # first tick measures from the default prev_position 0; the cycle restarts at the slice END going backwards
    assert deltas(a, 0.75, 4) == [(2.0, 3.0, 0.0), (-0.75, 0.0, 0.0), (-0.75, 0.0, 0.0), (-0.75, 0.0, 0.0)]


def test_speed_zero_and_ignore_flags():
    a = walk(speed=0.0, time_position=1.0)
    a.set_root_motion_settings(node=1, ignore_y=True)
    assert deltas(a, 0.5, 2) == [(1.0, 0.0, 0.0), (0.0, 0.0, 0.0)]
    assert tuple(a.pose_val[0][:3]) == (0.0, 3.0, 0.0)  # y ignored: kept from the pose (3), x reset to the start
    b = walk()
    b.set_root_motion_settings(node=1, ignore_x=True, ignore_z=True)
    assert deltas(b, 0.5, 2)[1] == (0.0, 0.0, 0.0)
    assert float(b.pose_val[0][0]) == 0.5  # x kept from the pose


def test_first_position_track_on_another_node():
    # the cycle values come from the animation's FIRST Position track, here node 2's (x = 2t)
    t, k = keys_tracks([(2, ob.BIND_POSITION, ob.TV_VECTOR3, [[(0.0, 0.0, LIN), (2.0, 4.0, LIN)], [(0.0, 0.0, CONST)], [(0.0, 0.0, CONST)]]),
                        (1, ob.BIND_POSITION, ob.TV_VECTOR3, RAMP_X)])
    a = rmo.Animation(t, k, speed=1.0, looped=True, time_slice=(0.0, 2.0))
    a.set_root_motion_settings(node=1)
    d = deltas(a, 0.75, 4)
    # tick 3 wraps: remainder = fetch_first(2) - pose = 4 - 1.5; tick 4: (0.25 - fetch_first(0)) + 2.5
    assert d[3] == (2.75, 0.0, 0.0)
    assert tuple(a.pose_val[1][:3]) == (0.0, 0.0, 0.0)  # reset to node 2's value at the slice start


def test_disabled_or_missing_root_track_gives_default_motion():
    a = walk()
    a.set_track_enabled(0, False)
    a.set_root_motion_settings(node=1)
    a.tick(0.5)
    assert a.root_motion is not None and a.root_motion.delta_position == rmo.ZERO3 and a.root_motion.delta_rotation == rmo.IDENTITY
    b = walk()
    b.set_root_motion_settings(node=7)  # nothing animates node 7
    b.tick(0.5)
    assert b.root_motion.delta_position == rmo.ZERO3


def test_settings_set_mid_play_and_removed():
    a = walk()
    a.tick(0.5)
    a.tick(0.5)
    assert a.root_motion is None
    a.set_root_motion_settings(node=1)
    assert deltas(a, 0.5, 2) == [(1.0, 3.0, 0.0), (0.5, 0.0, 0.0)]  # first from prev_position 0
    a.set_root_motion_settings(None)
    a.tick(0.5)
    assert a.root_motion.delta_position == (f32(0.5), f32(0), f32(0))  # stays as it was
    assert float(a.pose_val[0][0]) == 2.0  # and the pose at t = 2 is no longer reset


def test_rotation_remainder_and_ignore_rotations():
    half = float(np.float32(np.sqrt(0.5)))
    rot = [[(0.0, 0.0, CONST)], [(0.0, 0.0, CONST)], [(0.0, 0.0, LIN), (2.0, half, LIN)], [(0.0, 1.0, LIN), (2.0, half, LIN)]]
    t, k = keys_tracks([(1, ob.BIND_ROTATION, ob.TV_QUAT, rot)])
    a = rmo.Animation(t, k, speed=1.0, looped=True, time_slice=(0.0, 2.0))
    a.set_root_motion_settings(node=1)
    for _ in range(3):
        a.tick(0.75)
    assert a.root_motion.rotation_remainder is not None  # the wrap
    q = np.array(a.root_motion.delta_rotation, np.float64)
    assert abs(np.linalg.norm(q) - 1) < 1e-6 and q[3] > 0.9
    assert tuple(a.pose_val[0]) == (0.0, 0.0, 0.0, 1.0)  # reset to the slice start's rotation
    b = rmo.Animation(t, k, speed=1.0, looped=True, time_slice=(0.0, 2.0))
    b.set_root_motion_settings(node=1, ignore_rotations=True)
    b.tick(0.75)
    b.tick(0.75)
    assert b.root_motion.delta_rotation == rmo.IDENTITY and float(b.pose_val[0][2]) != 0.0


def events(a, dt, n):
    out = []
    for _ in range(n):
        a.tick(dt)
        out.append(a.take_events())
    return out


def test_signals_at_cur_at_new_and_past_the_end():
    a = walk()
    for tm in (0.0, 0.5, 2.5):
        a.add_signal(tm)
    a.add_signal(1.0, enabled=False)
    # ticks: 0 -> 0.5 (fires 0.5; 0.0 sits at cur: no), 0.5 -> 1.0, 1.0 -> 1.5, 1.5 -> 2.0, 2.0 -> 2.5 (wraps; 2.5 fires)
    assert events(a, 0.5, 5) == [[1], [], [], [], [2]]


def test_negative_speed_capacity_binds_only_backwards():
    a = walk(speed=-1.0, time_position=2.0)
    for tm in (1.75, 1.5, 1.25):
        a.add_signal(tm)
    a.max_event_capacity = 2
    a.tick(1.0)
    assert a.take_events() == [0, 1]  # the third would exceed the capacity
    b = walk(speed=1.0)
    for tm in (0.25, 0.5, 0.75):
        b.add_signal(tm)
    b.max_event_capacity = 1
    b.tick(1.0)
    assert b.take_events() == [0, 1, 2]  # speed >= 0: no limit
    c = walk(speed=float("nan"))
    c.add_signal(0.0)
    c.add_signal(1.0)
    c.tick(0.5)
    assert c.take_events() == []


def test_group_running_blends():
    srcs = [walk(), walk(), walk(time_position=1.0)]
    srcs[0].set_root_motion_settings(node=1)
    srcs[2].set_root_motion_settings(node=1)  # srcs[1] has no settings: it hands on None = default
    for w in ([0.0, 0.5, 1.0], [2.0, 0.5, 0.5]):
        g = rmo.BlendGroup([walk(), walk(), walk(time_position=1.0)], w)
        for a, s in zip(g.sources, srcs):
            a.root_motion_settings = s.root_motion_settings
        out = np.zeros(3, np.float32)
        fin = np.zeros(3, np.float32)
        og = ob.Graph.build(np.array([0xFFFFFFFF, 0], np.uint32))
        tr = (ob.Transform * 2)()
        for _ in range(4):
            g.update(0.5, og, tr)
            for a, wi in zip(g.sources, g.weights):  # lerp a * (1 - w) + b * w, the running fold from last frame's value
                d = np.array(a.root_motion.delta_position if a.root_motion is not None else rmo.ZERO3, np.float32)
                out = out * (f32(1) - wi) + d * wi
            fin = fin * (f32(1) - f32(1)) + out * f32(1)
            assert (np.array(g.output_root_motion.delta_position, np.float32) == out).all()
            assert (np.array(g.root_motion.delta_position, np.float32) == fin).all()
        g.sources[0].set_enabled(False)  # a disabled source hands on its stale motion
        stale = g.sources[0].root_motion.delta_position
        g.update(0.5, og, tr)
        assert g.sources[0].root_motion.delta_position == stale


def test_without_features_tick_is_the_c_oracles():
    rng = np.random.default_rng(3)
    spec = []
    for node in range(1, 6):
        spec.append((node, ob.BIND_POSITION, ob.TV_VECTOR3, [[(float(l), float(rng.uniform(-2, 2)), int(rng.integers(0, 3)))
                                                                for l in sorted(rng.integers(0, 8, 4) * 0.25)] for _ in range(3)]))
    t, k = keys_tracks(spec)
    kw = dict(speed=1.5, looped=True, time_slice=(0.0, 1.75), time_position=0.25)
    a, b = rmo.Animation(t, k, **kw), ob.Animation(t, k, **kw)
    og_a = ob.Graph.build(np.array([0xFFFFFFFF, 0, 0, 0, 0, 0], np.uint32))
    og_b = ob.Graph.build(np.array([0xFFFFFFFF, 0, 0, 0, 0, 0], np.uint32))
    tr_a, tr_b = (ob.Transform * 6)(), (ob.Transform * 6)()
    for i in range(6):
        ob.lib().orc_transform_identity(C.byref(tr_a[i]))
        ob.lib().orc_transform_identity(C.byref(tr_b[i]))
    for dt in (0.125, 0.3, 0.125, 0.7, 0.25, 0.125):
        rmo.update_animations([a], dt, og_a, tr_a)
        ob.update_animations([b], dt, og_b, tr_b)
        og_a.update()
        og_b.update()
        assert np.float32(a.time_position).tobytes() == np.float32(b.time_position).tobytes()
        for i in range(6):
            assert bytes(tr_a[i]) == bytes(tr_b[i])
        assert og_a.global_transforms().tobytes() == og_b.global_transforms().tobytes()
