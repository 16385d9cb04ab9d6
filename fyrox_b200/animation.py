"""Host mirror of the reference's animation data model (fyrox-math/src/curve.rs, fyrox-animation/src/{track,container,
lib}.rs) — the objects a Fyrox host owns — and the flattening of an ``Animation`` into the ``fyx_anim_track`` /
``fyx_curve_key`` arrays ``fyx_anim_add`` takes (INTEGRATION.md S0).  Same names and argument meaning as the reference.

Nothing here samples a curve: sampling, pose application and time advance are the device's job (``Context.animate``).
This module is host logic only and runs without a GPU (``tests/test_host_mirror_cpu.py`` pins it with the reference's
own curve tests and checks the flattened form against the oracle).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import numpy as np

from ._lib import (BIND_POSITION, BIND_ROTATION, BIND_SCALE, KEY_CONSTANT, KEY_CUBIC, KEY_LINEAR, TV_QUAT, TV_QUAT_EULER, TV_REAL, TV_VECTOR2,
                   TV_VECTOR3, TV_VECTOR4)

KEY_DTYPE = np.dtype([("location", "<f4"), ("value", "<f4"), ("kind", "<u4"), ("left_tangent", "<f4"), ("right_tangent", "<f4")])
TRACK_DTYPE = np.dtype([("target_node", "<u4"), ("binding", "<u4"), ("value_kind", "<u4"), ("enabled", "<u4"), ("n_curves", "<u4"),
                        ("first_key", "<u4", 4), ("n_keys", "<u4", 4)])

_f32 = np.float32


@dataclass(frozen=True)
class CurveKeyKind:
    """fyrox-math/src/curve.rs:33-55.  ``kind`` is FYX_KEY_*; tangents are tan(angle) and only meaningful for Cubic."""

    kind: int = KEY_CONSTANT
    left_tangent: float = 0.0
    right_tangent: float = 0.0

    @staticmethod
    def constant() -> "CurveKeyKind":
        return CurveKeyKind(KEY_CONSTANT)

    @staticmethod
    def linear() -> "CurveKeyKind":
        return CurveKeyKind(KEY_LINEAR)

    @staticmethod
    def cubic(left_tangent: float, right_tangent: float) -> "CurveKeyKind":
        return CurveKeyKind(KEY_CUBIC, float(_f32(left_tangent)), float(_f32(right_tangent)))

    @staticmethod
    def new_cubic(left_angle_radians: float, right_angle_radians: float) -> "CurveKeyKind":
        """curve.rs:47-54: tangents are the tan() of the angles (f32 tan of the platform, as in the reference)."""
        return CurveKeyKind(KEY_CUBIC, float(_f32(math.tan(_f32(left_angle_radians)))), float(_f32(math.tan(_f32(right_angle_radians)))))


@dataclass
class CurveKey:
    """curve.rs:57-75"""

    location: float = 0.0
    value: float = 0.0
    kind: CurveKeyKind = field(default_factory=CurveKeyKind)

    def __post_init__(self):
        self.location = float(_f32(self.location))
        self.value = float(_f32(self.value))


class Curve:
    """curve.rs:150-255 — keys are kept sorted by location; equal locations keep their insertion order
    (Rust's ``sort_by`` is stable, ``add_key`` inserts before the first key that is not smaller)."""

    def __init__(self, keys: Optional[List[CurveKey]] = None):
        self.keys: List[CurveKey] = []
        self.name = ""
        if keys:
            self.keys = sorted(keys, key=lambda k: k.location)  # From<Vec<CurveKey>>: stable sort by location

    def clear(self):
        self.keys.clear()

    def is_empty(self) -> bool:
        return not self.keys

    def add_key(self, new_key: CurveKey):
        pos = 0  # partition_point(|k| k.location < new_key.location)
        while pos < len(self.keys) and self.keys[pos].location < new_key.location:
            pos += 1
        self.keys.insert(pos, new_key)

    def move_key(self, key_id: int, location: float):
        if 0 <= key_id < len(self.keys):
            self.keys[key_id].location = float(_f32(location))
            self.keys.sort(key=lambda k: k.location)

    def max_location(self) -> float:
        return self.keys[-1].location if self.keys else 0.0

    def keys_values(self) -> List[float]:
        return [k.value for k in self.keys]


class TrackValueKind:
    """fyrox-animation/src/container.rs:41-76"""

    Real, Vector2, Vector3, Vector4, UnitQuaternionEuler, UnitQuaternion = TV_REAL, TV_VECTOR2, TV_VECTOR3, TV_VECTOR4, TV_QUAT_EULER, TV_QUAT

    @staticmethod
    def components_count(kind: int) -> int:
        return {TV_REAL: 1, TV_VECTOR2: 2, TV_VECTOR3: 3, TV_VECTOR4: 4, TV_QUAT_EULER: 3, TV_QUAT: 4}[kind]


class ValueBinding:
    """fyrox-animation/src/value.rs:358-374 (property bindings are not supported on the device)"""

    Position, Scale, Rotation = BIND_POSITION, BIND_SCALE, BIND_ROTATION


class TrackDataContainer:
    """container.rs:99-160: `components_count` default curves for the kind"""

    def __init__(self, kind: int = TrackValueKind.Vector3):
        self.kind = kind
        self.curves: List[Curve] = [Curve() for _ in range(TrackValueKind.components_count(kind))]

    def add_curve(self, curve: Curve):
        self.curves.append(curve)

    def curve_mut(self, index: int) -> Optional[Curve]:
        return self.curves[index] if 0 <= index < len(self.curves) else None

    def time_length(self) -> float:
        """container.rs:303-312: the right-most key of any curve"""
        length = 0.0
        for c in self.curves:
            if c.max_location() > length:
                length = c.max_location()
        return length


class Track:
    """fyrox-animation/src/track.rs:95-205"""

    _next_id = 0

    def __init__(self, container: Optional[TrackDataContainer] = None, binding: int = ValueBinding.Position):
        self.frames = container if container is not None else TrackDataContainer()
        self.binding = binding
        Track._next_id += 1
        self.id = Track._next_id  # stands for the Uuid

    @staticmethod
    def new_position() -> "Track":
        return Track(TrackDataContainer(TrackValueKind.Vector3), ValueBinding.Position)

    @staticmethod
    def new_rotation() -> "Track":
        return Track(TrackDataContainer(TrackValueKind.UnitQuaternionEuler), ValueBinding.Rotation)  # track.rs:139-145

    @staticmethod
    def new_scale() -> "Track":
        return Track(TrackDataContainer(TrackValueKind.Vector3), ValueBinding.Scale)

    def data_container(self) -> TrackDataContainer:
        return self.frames

    def time_length(self) -> float:
        return self.frames.time_length()


@dataclass
class TrackBinding:
    """track.rs:36-93: target node (index) and the enabled switch"""

    target: int
    enabled: bool = True


@dataclass
class AnimationSignal:
    """fyrox-animation/src/signal.rs:44-74: `id` stands for the Uuid; events name the signal by it."""

    id: int = 0
    name: str = ""
    time: float = 0.0
    enabled: bool = True


@dataclass
class AnimationEvent:
    """lib.rs: the signal_id and name of the signal that fired."""

    signal_id: int
    name: str


@dataclass
class RootMotionSettings:
    """lib.rs:305-319"""

    node: int = 0
    ignore_x_movement: bool = False
    ignore_y_movement: bool = False
    ignore_z_movement: bool = False
    ignore_rotations: bool = False


@dataclass
class RootMotion:
    """lib.rs:324-336, the public part: what Animation::root_motion() shows a game."""

    delta_position: Tuple[float, float, float] = (0.0, 0.0, 0.0)
    delta_rotation: Tuple[float, float, float, float] = (0.0, 0.0, 0.0, 1.0)  # (i, j, k, w)


class Animation:
    """fyrox-animation/src/lib.rs:269-496, 755-790, 922-945 — the data and switches of one animation; defaults as
    Animation::default (speed 1, looped, enabled, empty time slice)."""

    def __init__(self, name: str = ""):
        self.name = name
        self.tracks: List[Track] = []  # AnimationTracksData::tracks
        self.track_bindings: Dict[int, TrackBinding] = {}
        self.speed = 1.0
        self.time_position = 0.0
        self.enabled = True
        self.looped = True
        self.time_slice: Tuple[float, float] = (0.0, 0.0)
        self.signals: List[AnimationSignal] = []
        self.max_event_capacity = 32
        self.events: List[AnimationEvent] = []  # filled by AnimationContainer.fetch_events from the device
        self.root_motion_settings: Optional[RootMotionSettings] = None
        self._root_motion: Optional[RootMotion] = None  # set by AnimationContainer.fetch_root_motions

    def add_signal(self, signal: AnimationSignal) -> AnimationSignal:
        self.signals.append(signal)
        return signal

    def set_max_event_capacity(self, capacity: int):
        self.max_event_capacity = int(capacity)

    def pop_event(self) -> Optional[AnimationEvent]:
        return self.events.pop(0) if self.events else None

    def take_events(self) -> List[AnimationEvent]:
        ev, self.events = self.events, []
        return ev

    def set_root_motion_settings(self, settings: Optional[RootMotionSettings]):
        self.root_motion_settings = settings

    def root_motion_settings_ref(self) -> Optional[RootMotionSettings]:
        return self.root_motion_settings

    def root_motion(self) -> Optional[RootMotion]:
        return self._root_motion

    def add_track_with_binding(self, binding: TrackBinding, track: Track):
        self.tracks.append(track)
        self.track_bindings[track.id] = binding

    def set_time_slice(self, start: float, end: float):
        assert start <= end  # lib.rs:446
        self.time_slice = (float(_f32(start)), float(_f32(end)))

    def fit_length_to_content(self):
        """lib.rs:410-421"""
        start, end = 0.0, self.time_slice[1]
        for t in self.tracks:
            if t.time_length() > end:
                end = t.time_length()
        self.time_slice = (start, end)

    def set_speed(self, speed: float):
        self.speed = float(speed)

    def set_loop(self, looped: bool):
        self.looped = bool(looped)

    def set_enabled(self, enabled: bool):
        self.enabled = bool(enabled)

    def flatten(self):
        """(tracks TRACK_DTYPE[n], keys KEY_DTYPE[m], kwargs for Context.anim_add): tracks in AnimationTracksData order; a
        track without a binding is left out exactly like update_pose skips it (lib.rs:903-905)."""
        tracks, keys = [], []
        for t in self.tracks:
            b = self.track_bindings.get(t.id)
            if b is None:
                continue
            rec = np.zeros((), TRACK_DTYPE)
            curves = t.frames.curves[:4]
            rec["target_node"], rec["binding"], rec["value_kind"] = b.target, t.binding, t.frames.kind
            rec["enabled"], rec["n_curves"] = int(b.enabled), len(curves)
            for c, curve in enumerate(curves):
                rec["first_key"][c], rec["n_keys"][c] = len(keys), len(curve.keys)
                for k in curve.keys:
                    keys.append((k.location, k.value, k.kind.kind, k.kind.left_tangent, k.kind.right_tangent))
            tracks.append(rec)
        ta = np.array(tracks, TRACK_DTYPE) if tracks else np.zeros(0, TRACK_DTYPE)
        ka = np.zeros(len(keys), KEY_DTYPE)
        for i, r in enumerate(keys):
            ka[i] = r
        kw = dict(speed=self.speed, looped=self.looped, time_slice=self.time_slice, time_position=self.time_position, enabled=self.enabled)
        return ta, ka, kw


class AnimationContainer:
    """lib.rs:947-1100 reduced to what the device needs: animations in pool order; ``upload`` hands them to a Context
    in that order (the order update_animations walks them) and returns the device ids."""

    def __init__(self):
        self.animations: List[Animation] = []

    def add(self, animation: Animation) -> int:
        self.animations.append(animation)
        return len(self.animations) - 1

    def upload(self, ctx) -> List[int]:
        """Also hands each animation's signals, event capacity and root-motion settings to the device."""
        ids = []
        for a in self.animations:
            t, k, kw = a.flatten()
            i = ctx.anim_add(t, k, **kw)
            if a.signals:
                ctx.anim_set_signals(i, [(s.time, s.enabled) for s in a.signals])
            if a.max_event_capacity != 32:
                ctx.anim_set_max_event_capacity(i, a.max_event_capacity)
            s = a.root_motion_settings
            if s is not None:
                ctx.anim_set_root_motion(i, s.node, s.ignore_x_movement, s.ignore_y_movement, s.ignore_z_movement, s.ignore_rotations)
            ids.append(i)
        return ids

    def fetch_events(self, ctx, ids: List[int]):
        """Drain the device's events into each animation's queue (then pop_event / take_events), mapping the signal index
        back to the signal's id and name.  The drain covers every animation of the context: events of animations that are
        not in `ids` (another container's) are dropped.  Returns the number of events the device dropped because a store
        was full."""
        by_id = {d: a for d, a in zip(ids, self.animations)}
        ev, lost = ctx.anim_take_events()
        for anim, sig in ev.tolist():
            a = by_id.get(anim)
            if a is not None:
                s = a.signals[sig]
                a.events.append(AnimationEvent(s.id, s.name))
        return lost

    def fetch_root_motions(self, ctx, ids: List[int]):
        """Animation::root_motion() of every animation, read back from the device."""
        if not ids:
            return
        rm = ctx.anim_root_motions(min(ids), max(ids) - min(ids) + 1)
        for d, a in zip(ids, self.animations):
            r = rm[d - min(ids)]
            a._root_motion = RootMotion(tuple(float(x) for x in r["delta_position"]), tuple(float(x) for x in r["delta_rotation"])) \
                if r["present"] else None
