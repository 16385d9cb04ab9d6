"""CPU restatement of Animation::tick with signals and root motion (fyrox-animation/src/lib.rs:471-661, signal.rs), of
the pose application that follows it (AnimationContainer::update_animations, fyrox-impl/src/scene/animation/mod.rs:83-88,
147-179) and of the one-layer, one-state blend machine over PlayAnimation sources with its two running root-motion
blends (machine/mod.rs:344-385, machine/node/blend.rs:136-166, machine/node/play.rs:84-100, pose.rs:41-101).

Test infrastructure only.  The pieces the C oracle already pins are called from it: TrackDataContainer::fetch
(orc_track_fetch), wrapf (orc_wrapf), TrackValue::blend_with (orc_track_value_blend).  Everything else is f32 arithmetic
in the reference's operation order; the quaternion product is nalgebra's, as in fyrox_anim_oracle.c.  With no signals and
no root-motion settings, `tick` is the C oracle's tick (tests/test_anim_root_motion_cpu.py checks that bit for bit).
"""
from __future__ import annotations

import ctypes as C
from collections import deque

import numpy as np

import oracle_binding as ob

f32 = np.float32
IDENTITY = (f32(0), f32(0), f32(0), f32(1))
ZERO3 = (f32(0), f32(0), f32(0))


def quat_mul(a, b):
    """nalgebra's a * b, components (i, j, k, w)."""
    w = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2]
    i = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1]
    j = a[3] * b[1] - a[0] * b[2] + a[1] * b[3] + a[2] * b[0]
    k = a[3] * b[2] + a[0] * b[1] - a[1] * b[0] + a[2] * b[3]
    return (f32(i), f32(j), f32(k), f32(w))


def quat_inverse(q):
    """UnitQuaternion::inverse = the conjugate."""
    return (-q[0], -q[1], -q[2], q[3])


def blend(a, b, w, is_quat):
    """TrackValue::blend_with / RootMotion::blend_with: lerp, or the shortest-way nlerp (value.rs:449-454)."""
    x = np.array(list(a) + [0.0] * (4 - len(a)), np.float32)
    y = np.array(list(b) + [0.0] * (4 - len(b)), np.float32)
    ob.lib().orc_track_value_blend(int(is_quat), ob.fp(x), ob.fp(y), float(w))
    return tuple(f32(v) for v in (x if is_quat else x[:3]))


class RootMotion:
    """lib.rs:324-336"""

    def __init__(self):
        self.delta_position = ZERO3
        self.delta_rotation = IDENTITY
        self.prev_position = ZERO3
        self.position_offset_remainder = None
        self.prev_rotation = IDENTITY
        self.rotation_remainder = None

    def copy(self):
        r = RootMotion()
        r.__dict__.update(self.__dict__)
        return r

    def blend_with(self, other: "RootMotion", weight):
        self.delta_position = blend(self.delta_position, other.delta_position, weight, False)
        self.delta_rotation = blend(self.delta_rotation, other.delta_rotation, weight, True)


class Animation:
    """Animation<Handle<Node>>: tracks (TRACK_DTYPE) over one key array (KEY_DTYPE); defaults as Animation::default."""

    def __init__(self, tracks, keys, speed=1.0, looped=True, time_slice=(0.0, 0.0), time_position=0.0, enabled=True):
        self.tracks = np.ascontiguousarray(tracks, dtype=ob.TRACK_DTYPE).copy()
        self.keys = np.ascontiguousarray(keys, dtype=ob.KEY_DTYPE)
        self.hints = np.zeros((len(self.tracks), 4), np.uint32)
        self.pose_val = np.zeros((len(self.tracks), 4), np.float32)
        self.pose_ok = np.zeros(len(self.tracks), bool)
        self.speed, self.looped, self.enabled = f32(speed), bool(looped), bool(enabled)
        self.time_slice = (f32(time_slice[0]), f32(time_slice[1]))
        self.time_position = f32(0)
        self.set_time_position(time_position)
        self.signals = []  # [time, enabled] in signal order
        self.events = deque()
        self.max_event_capacity = 32
        self.root_motion_settings = None  # dict(node, ignore_x, ignore_y, ignore_z, ignore_rotations)
        self.root_motion = None

    # ---- the reference's setters ----
    def set_time_position(self, t):
        t = f32(t)
        if self.looped:
            self.time_position = f32(ob.lib().orc_wrapf(float(t), float(self.time_slice[0]), float(self.time_slice[1])))
        else:  # f32::clamp
            x = t
            if x < self.time_slice[0]:
                x = self.time_slice[0]
            if x > self.time_slice[1]:
                x = self.time_slice[1]
            self.time_position = f32(x)

    def set_speed(self, s):
        self.speed = f32(s)

    def set_enabled(self, e):
        self.enabled = bool(e)

    def set_track_enabled(self, t, e):
        self.tracks[t]["enabled"] = int(bool(e))

    def add_signal(self, time, enabled=True):
        self.signals.append([f32(time), bool(enabled)])

    def set_root_motion_settings(self, node=None, ignore_x=False, ignore_y=False, ignore_z=False, ignore_rotations=False):
        self.root_motion_settings = None if node is None else dict(node=int(node), ignore_x=ignore_x, ignore_y=ignore_y, ignore_z=ignore_z,
                                                                   ignore_rotations=ignore_rotations)

    def take_events(self):
        ev, self.events = list(self.events), deque()
        return ev

    # ---- tick ----
    def _fetch(self, ti, time, hints):
        out = np.zeros(4, np.float32)
        ok = ob.lib().orc_track_fetch(self.tracks[ti:ti + 1].ctypes.data_as(C.c_void_p), self.keys.ctypes.data_as(C.c_void_p), float(time),
                                      hints.ctypes.data_as(C.POINTER(C.c_uint32)), ob.fp(out))
        return bool(ok), out

    def update_pose(self):
        """lib.rs:895-914"""
        for ti in range(len(self.tracks)):
            self.pose_ok[ti] = False
            if not self.tracks[ti]["enabled"]:
                continue
            h = np.ascontiguousarray(self.hints[ti])
            ok, v = self._fetch(ti, self.time_position, h)
            self.hints[ti] = h
            if ok:
                self.pose_ok[ti], self.pose_val[ti] = True, v

    def _fetch_first(self, binding, time):
        """fetch_position_at_time / fetch_rotation_at_time (lib.rs:505-533)"""
        rotation = binding == ob.BIND_ROTATION
        for ti in range(len(self.tracks)):
            if self.tracks[ti]["binding"] != binding:
                continue
            kind = self.tracks[ti]["value_kind"]
            ok, v = self._fetch(ti, time, np.zeros(4, np.uint32))
            if ok and (kind in (ob.TV_QUAT, ob.TV_QUAT_EULER) if rotation else kind == ob.TV_VECTOR3):
                return tuple(f32(x) for x in (v if rotation else v[:3]))
            break
        return IDENTITY if rotation else ZERO3

    def tick(self, dt):
        """lib.rs:471-496"""
        self.update_pose()
        cur = self.time_position
        new = f32(cur + f32(dt) * self.speed)
        for i, (time, enabled) in enumerate(self.signals):
            if not enabled:
                continue
            if (self.speed >= 0 and (cur < time and new >= time)) or \
                    (self.speed < 0 and (cur > time and new <= time) and len(self.events) < self.max_event_capacity):
                self.events.append(i)
        self.set_time_position(new)
        self.update_root_motion(cur)

    def update_root_motion(self, prev_time):
        """lib.rs:498-661"""
        st = self.root_motion_settings
        if st is None:
            return
        prev = self.root_motion.copy() if self.root_motion is not None else RootMotion()
        new_cycle = self.looped and ((self.speed > 0 and self.time_position < prev_time) or (self.speed < 0 and self.time_position > prev_time))
        cycle_start = self.time_slice[0] if self.speed > 0 else self.time_slice[1]
        cycle_end = self.time_slice[1] if self.speed > 0 else self.time_slice[0]
        rm = RootMotion()
        for ti in range(len(self.tracks)):  # the root's NodePose values, in push order
            t = self.tracks[ti]
            if not self.pose_ok[ti] or t["target_node"] != st["node"]:
                continue
            if t["binding"] == ob.BIND_POSITION and t["value_kind"] == ob.TV_VECTOR3:
                p = tuple(f32(x) for x in self.pose_val[ti][:3])
                if new_cycle:
                    rm.prev_position = self._fetch_first(ob.BIND_POSITION, cycle_start)
                    e = self._fetch_first(ob.BIND_POSITION, cycle_end)
                    rm.position_offset_remainder = tuple(f32(e[k] - p[k]) for k in range(3))
                else:
                    rm.prev_position = p
                rem = prev.position_offset_remainder if prev.position_offset_remainder is not None else ZERO3
                delta = tuple(f32(f32(p[k] - prev.prev_position[k]) + rem[k]) for k in range(3))
                ign = (st["ignore_x"], st["ignore_y"], st["ignore_z"])
                rm.delta_position = tuple(f32(0) if ign[k] else delta[k] for k in range(3))
                start = self._fetch_first(ob.BIND_POSITION, self.time_slice[0])
                self.pose_val[ti][:3] = [p[k] if ign[k] else start[k] for k in range(3)]
            elif t["binding"] == ob.BIND_ROTATION and t["value_kind"] in (ob.TV_QUAT, ob.TV_QUAT_EULER) and not st["ignore_rotations"]:
                q = tuple(f32(x) for x in self.pose_val[ti])
                if new_cycle:
                    rm.prev_rotation = self._fetch_first(ob.BIND_ROTATION, cycle_start)
                    rm.rotation_remainder = quat_mul(quat_inverse(self._fetch_first(ob.BIND_ROTATION, cycle_end)), q)
                else:
                    rm.prev_rotation = q
                rem = prev.rotation_remainder if prev.rotation_remainder is not None else IDENTITY
                rm.delta_rotation = quat_mul(rem, quat_mul(quat_inverse(prev.prev_rotation), q))
                self.pose_val[ti] = self._fetch_first(ob.BIND_ROTATION, self.time_slice[0])
        self.root_motion = rm


# ---- pose application (scene/animation/mod.rs:147-179 through scene/transform.rs:202-262) ----
def _apply_value(binding, is_quat, is_vec3, v, n, graph, transforms, dirty, touched):
    if n >= len(transforms) or not graph.L.orc_node_is_alive(graph.h, n):
        return
    tr = transforms[n]
    if binding == ob.BIND_POSITION and is_vec3:
        touched[n] = 1
        if dirty[n] or tuple(tr.local_position) != tuple(v[:3]):
            tr.local_position[:] = [float(x) for x in v[:3]]
            dirty[n] = 1
    elif binding == ob.BIND_SCALE and is_vec3:
        touched[n] = 1
        if dirty[n] or tuple(tr.local_scale) != tuple(v[:3]):
            tr.local_scale[:] = [float(x) for x in v[:3]]
            dirty[n] = 1
    elif binding == ob.BIND_ROTATION and is_quat:
        touched[n] = 1
        cur = np.array(tr.local_rotation, np.float32)
        vv = np.asarray(v[:4], np.float32)
        if dirty[n] or not ((cur == vv).all() or (cur == -vv).all()):
            tr.local_rotation[:] = [float(x) for x in vv]
            dirty[n] = 1


def _is_quat(kind):
    return kind in (ob.TV_QUAT, ob.TV_QUAT_EULER)


def _frame(graph, transforms):
    n = len(transforms)
    graph.frame_dirty(n)
    return graph._frame_dirty, np.zeros(max(n, 1), np.uint8)


def _refresh(graph, transforms, touched):
    for k in np.nonzero(touched[:len(transforms)])[0]:
        graph.L.orc_node_set_local_transform(graph.h, int(k), C.byref(transforms[int(k)]))


def update_animations(anims, dt, graph, transforms):
    """AnimationContainer::update_animations: every enabled animation ticks and applies its pose."""
    dirty, touched = _frame(graph, transforms)
    for a in anims:
        if a.enabled:
            a.tick(dt)
            for ti in range(len(a.tracks)):
                if a.pose_ok[ti]:
                    t = a.tracks[ti]
                    _apply_value(t["binding"], _is_quat(t["value_kind"]), t["value_kind"] == ob.TV_VECTOR3, a.pose_val[ti], int(t["target_node"]),
                                 graph, transforms, dirty, touched)
    _refresh(graph, transforms, touched)


class BlendGroup:
    """One Machine with one layer and one state whose root is BlendAnimations over PlayAnimation sources with constant
    weights.  `output_root_motion` is BlendAnimations' output pose's and `root_motion` the machine's final pose's: neither
    is cleared by AnimationPose::reset."""

    def __init__(self, sources, weights):
        self.sources, self.weights = list(sources), [f32(w) for w in weights]
        self.output_root_motion = None
        self.root_motion = None

    def update(self, dt, graph, transforms):
        for a in self.sources:
            if a.enabled:
                a.tick(dt)
        out = {}  # node -> [[binding, is_quat, is_vec3, value]] (NodePose values)
        for a, w in zip(self.sources, self.weights):
            src = {}
            for ti in range(len(a.tracks)):
                if not a.pose_ok[ti]:
                    continue
                t = a.tracks[ti]
                src.setdefault(int(t["target_node"]), []).append([int(t["binding"]), _is_quat(t["value_kind"]), t["value_kind"] == ob.TV_VECTOR3,
                                                                   a.pose_val[ti].copy()])
            for node, vals in src.items():
                if node >= len(transforms):
                    continue
                if node not in out or not out[node]:
                    out[node] = [[b, q, v3, val.copy()] for b, q, v3, val in vals]
                    continue
                for ov in out[node]:
                    for sv in vals:
                        if sv[0] == ov[0]:
                            if ov[1] and sv[1]:
                                ov[3] = np.array(blend(ov[3], sv[3], w, True), np.float32)
                            elif ov[2] and sv[2]:
                                ov[3] = np.array(list(blend(ov[3][:3], sv[3][:3], w, False)) + [0.0], np.float32)
                            break
            # the running root-motion blend (pose.rs:96-100, play.rs:96-97)
            if self.output_root_motion is None:
                self.output_root_motion = RootMotion()
            self.output_root_motion.blend_with(a.root_motion if a.root_motion is not None else RootMotion(), w)
        if self.root_motion is None:
            self.root_motion = RootMotion()
        if self.output_root_motion is not None:  # the layer's clone, blended into the final pose with weight 1
            self.root_motion.blend_with(self.output_root_motion, 1.0)
        dirty, touched = _frame(graph, transforms)
        for node in sorted(out):
            for b, q, v3, val in out[node]:
                _apply_value(b, q, v3, val, node, graph, transforms, dirty, touched)
        _refresh(graph, transforms, touched)


def root_motion_record(rm):
    """(delta_position[3], delta_rotation[4], present) as fyx_anim_get_root_motions returns it."""
    if rm is None:
        return np.array([0, 0, 0], np.float32), np.array(IDENTITY, np.float32), 0
    return np.array(rm.delta_position, np.float32), np.array(rm.delta_rotation, np.float32), 1
