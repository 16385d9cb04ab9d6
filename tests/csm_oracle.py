"""Oracle of fyx_cull_shadow_casters_csm: the shadow-map loop of tests/shadow_oracle.py plus the cascaded shadow maps of the
directional lights (renderer/shadow/csm.rs:165-277, gated by renderer/light.rs:555-565), in f32 numpy over the C oracle's
primitives (orc_perspective, orc_mat4_mul, orc_mat4_transform_point, orc_orthographic,
orc_frustum_from_view_projection_matrix, orc_collect_lights, orc_from_graph).  Paths are relative to the Fyrox tree.

nalgebra and approx have no source in the reference tree, so three of their functions are restated here from their
documented definitions and are not pinned by a reference test: Matrix4::look_at_lh (Rotation3::face_towards inverted, then
applied to -eye), Matrix4::new_perspective with a general aspect (orc_perspective's order, m22 = 1 / tan(fov / 2) taken from
orc_perspective itself so that the platform's tanf gives it) and approx's relative_eq.  Matrix4::new_orthographic is the
oracle's orc_orthographic.

Every f32 operation below is one numpy float32 scalar operation: one rounding each, nothing contracted, in the
reference's order.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

import oracle_binding as ob
import shadow_oracle as so

f32 = np.float32
F32_EPSILON = so.F32_EPSILON
F32_MAX = f32(3.4028234663852886e38)
LIMIT = f32(10.0) * F32_EPSILON  # scene/camera.rs:90, 156
MIN_DEPTH_DELTA = F32_EPSILON * f32(2.0)  # shadow/csm.rs:202
PERSPECTIVE, ORTHOGRAPHIC = 0, 1
CSM_DEFAULT = (0, (5.0, 25.0, 64.0))  # FrustumSplitOptions::default(): Absolute { far_planes: [5, 25, 64] }


@dataclass
class CsmCamera:
    """What csm.rs reads from the camera: its projection (with fov or vertical_size), the projection's own z_near / z_far,
    Camera::view_matrix, the frame size (light.rs:767) and QualitySettings::csm_settings.enabled; plus the per-light
    FrustumSplitOptions {node: (relative, (s0, s1, s2))} (missing = CSM_DEFAULT)."""
    projection: int
    fov_or_vertical_size: float
    z_near: float
    z_far: float
    frame_size: tuple
    view_matrix: np.ndarray
    enabled: bool = True
    options: dict = field(default_factory=dict)


def relative_eq(a, b) -> bool:
    """approx's relative_eq!(a, b) for f32: epsilon = max_relative = f32::EPSILON."""
    a, b = f32(a), f32(b)
    if a == b:
        return True
    if np.isinf(a) or np.isinf(b):
        return False
    d = abs(a - b)
    if d <= F32_EPSILON:
        return True
    aa, ab = abs(a), abs(b)
    largest = ab if ab > aa else aa
    return bool(d <= largest * F32_EPSILON)


def m22_of(fov) -> np.float32:
    """1 / tan(fov / 2) as Perspective3::set_fovy computes it, through the C oracle's tanf."""
    return ob.perspective(1.0, float(f32(fov)), 1.0, 2.0)[5]


def perspective(m22, aspect, zn, zf):
    """Matrix4::new_perspective(aspect, fovy, zn, zf) with m22 = 1 / tan(fovy / 2) given (orc_perspective's order)."""
    m22, aspect, zn, zf = f32(m22), f32(aspect), f32(zn), f32(zf)
    out = np.zeros(16, f32)
    out[5] = m22
    out[0] = m22 / aspect
    out[10] = (zf + zn) / (zn - zf)
    out[14] = zf * zn * f32(2.0) / (zn - zf)
    out[11] = f32(-1.0)
    return out


def orthographic(l, r, b, t, zn, zf):
    out = np.empty(16, f32)
    ob.lib().orc_orthographic(*[float(f32(v)) for v in (l, r, b, t, zn, zf)], ob.fp(out))
    return out


def clamp_to_limit_signed(v):
    """scene/camera.rs:143-151."""
    v = f32(v)
    if v < 0.0 and -v < LIMIT:
        return -LIMIT
    if v >= 0.0 and v < LIMIT:
        return LIMIT
    return v


def projection_matrix(cam: CsmCamera, z_near, z_far):
    """Projection::with_z_near(z_near).with_z_far(z_far).matrix(frame_size) (scene/camera.rs:89-174)."""
    z_near, z_far = f32(z_near), f32(z_far)
    zn = np.fmin(z_far, z_near)  # f32::min / max: a NaN operand yields the other
    zf = np.fmax(z_far, z_near)
    if zf - zn < LIMIT:
        zf = zf + LIMIT
    aspect = np.fmax(f32(cam.frame_size[0]) / f32(cam.frame_size[1]), LIMIT)
    if cam.projection == PERSPECTIVE:
        return perspective(m22_of(cam.fov_or_vertical_size), aspect, zn, zf)
    vs = clamp_to_limit_signed(cam.fov_or_vertical_size)
    hs = clamp_to_limit_signed(aspect * vs)
    return orthographic(-hs, hs, -vs, vs, zn, zf)


def cross(a, b):
    return np.array([a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]], f32)


def look_at_lh(eye, target, up):
    """Matrix4::look_at_lh: rows s, u, f with f = normalize(target - eye), s = normalize(up x f), u = f x s; translation
    = rotation * (-eye)."""
    eye, target, up = (np.asarray(v, f32) for v in (eye, target, up))
    f = target - eye
    f = f / so.norm(f)
    s = cross(up, f)
    s = s / so.norm(s)
    u = cross(f, s)
    ne = -eye
    out = np.zeros(16, f32)
    out[0], out[4], out[8], out[12] = s[0], s[1], s[2], so.dot3(s, ne)
    out[1], out[5], out[9], out[13] = u[0], u[1], u[2], so.dot3(u, ne)
    out[2], out[6], out[10], out[14] = f[0], f[1], f[2], so.dot3(f, ne)
    out[15] = f32(1.0)
    return out


def transform_point(m, p):
    out = np.empty(3, f32)
    ob.lib().orc_mat4_transform_point(ob.fp(np.ascontiguousarray(m, f32)), ob.fp(np.ascontiguousarray(p, f32)), ob.fp(out))
    return out


def frustum_center(corners):
    """Frustum::center (fyrox-math/src/frustum.rs:197-202)."""
    acc = np.zeros(3, f32)
    for c in corners:
        acc = acc + c
    return acc * f32(0.125)


def z_values(cam: CsmCamera, options):
    """shadow/csm.rs:181-194."""
    relative, splits = options
    zn, zf = f32(cam.z_near), f32(cam.z_far)
    if relative:
        return [zn] + [zf * f32(s) for s in splits]
    return [zn] + [f32(s) for s in splits]


def cascade_depths(cam: CsmCamera, options, i):
    """(z_near, z_far) of cascade i, after the guard against relatively equal planes (shadow/csm.rs:195-205)."""
    zv = z_values(cam, options)
    z_near, z_far = zv[i], zv[i + 1]
    if relative_eq(z_far, z_near):
        z_far = z_far + MIN_DEPTH_DELTA * z_near
    return z_near, z_far


def slice_corners(cam: CsmCamera, z_near, z_far):
    """Corners of Frustum::from_view_projection_matrix(projection · view).unwrap_or_default() (shadow/csm.rs:207-219)."""
    view = np.asarray(cam.view_matrix, f32).reshape(16)
    fr = ob.frustum_from_vp(ob.mat4_mul(projection_matrix(cam, z_near, z_far), view)) or so.default_frustum()
    return ob.frustum_planes_corners(fr)[1]


def z_stretch(lo, hi):
    """shadow/csm.rs:235-246: z_mult = 10 pushes both depth bounds away from the light-space origin."""
    z_mult = f32(10.0)
    lo = lo * z_mult if lo < 0.0 else lo / z_mult
    hi = hi / z_mult if hi < 0.0 else hi * z_mult
    return lo, hi


def cascades(cam: CsmCamera, options, up_vector, look_vector):
    """The three cascades of one directional light: [(light view matrix, view_projection)] (shadow/csm.rs:170-249)."""
    light_direction = -so.try_normalize(up_vector, F32_EPSILON, (0.0, 1.0, 0.0))
    light_up = so.try_normalize(look_vector, F32_EPSILON, (0.0, 0.0, 1.0))
    out = []
    for i in range(3):
        corners = slice_corners(cam, *cascade_depths(cam, options, i))
        center = frustum_center(corners)
        v = look_at_lh(center + light_direction, center, light_up)
        mn = np.full(3, F32_MAX, f32)
        mx = np.full(3, -F32_MAX, f32)
        for c in corners:
            t = transform_point(v, c)
            for k in range(3):  # AxisAlignedBoundingBox::add_point
                if t[k] < mn[k]:
                    mn[k] = t[k]
                if t[k] > mx[k]:
                    mx[k] = t[k]
        mn[2], mx[2] = z_stretch(mn[2], mx[2])
        out.append((v, ob.mat4_mul(orthographic(mn[0], mx[0], mn[1], mx[1], mn[2], mx[2]), v)))
    return out


def directional_maps(og: ob.Graph, flags, camera: ob.Frustum, render_mask, light, local_scale, csm: CsmCamera):
    """The maps of one directional light of the camera's light list (light.rs:555-606 gating, then csm.rs)."""
    g = og.global_transform(light)
    position = g[12:15].astype(f32)
    up_vector, look_vector = g[4:7].astype(f32), g[8:11].astype(f32)
    shadows_enabled = bool(int(flags[light]) & so.NODE_CAST_SHADOWS) and bool(csm.enabled)
    scl = np.asarray(local_scale.get(light, (1.0, 1.0, 1.0)), f32)
    light_radius = f32(np.fmax(np.fmax(scl[0], scl[1]), scl[2])) * F32_MAX  # may be inf; a zero scale gives 0
    if not so.frustum_is_intersects_sphere(camera, position, light_radius) or not shadows_enabled:
        return []
    out = []
    for i, (v, vp) in enumerate(cascades(csm, csm.options.get(light, CSM_DEFAULT), up_vector, look_vector)):
        fr = ob.frustum_from_vp(vp) or so.default_frustum()
        vis = np.sort(og.from_graph(fr, render_mask, shadow_pass=True))
        out.append((light, 0, i, vp, vis))
    return out


def shadow_maps(og: ob.Graph, flags, camera: ob.Frustum, camera_translation, render_mask, settings, sources, local_scale, csm=None):
    """shadow_oracle.shadow_maps, plus the cascades of the directional lights when `csm` (a CsmCamera) is given, each light's
    maps in the light loop's pool order.  csm=None returns exactly what shadow_oracle.shadow_maps returns."""
    base = so.shadow_maps(og, flags, camera, camera_translation, render_mask, settings, sources, local_scale)
    if csm is None:
        return base
    by_light = {}
    for m in base:
        by_light.setdefault(m[0], []).append(m)
    out = []
    with np.errstate(all="ignore"):
        for light in og.collect_lights(camera):
            light = int(light)
            if light in sources and sources[light][0] == so.LIGHT_DIRECTIONAL:
                out += directional_maps(og, flags, camera, render_mask, light, local_scale, csm)
            else:
                out += by_light.get(light, [])
    return out


def cascade_views(og: ob.Graph, light, csm: CsmCamera):
    """The look_at_lh of each cascade of `light` (the observer's view matrix its instances are sorted by)."""
    g = og.global_transform(light)
    with np.errstate(all="ignore"):
        return [v for v, _ in cascades(csm, csm.options.get(light, CSM_DEFAULT), g[4:7].astype(f32), g[8:11].astype(f32))]

