"""Oracle of fyx_cull_shadow_casters: the shadow-map loop of the deferred light renderer, restated line by line in f32 numpy
on top of the C oracle's primitives (orc_look_at_rh, orc_perspective, orc_mat4_mul, orc_frustum_from_view_projection_matrix,
orc_collect_lights, orc_from_graph).  Paths are relative to the Fyrox tree.

Every f32 operation below is one numpy float32 scalar operation: one rounding each, nothing contracted, in the
reference's order.
"""
from __future__ import annotations

import numpy as np

import oracle_binding as ob

f32 = np.float32
FRAC_PI_2 = f32(1.57079632679489661923)
F32_EPSILON = f32(1.1920929e-07)

NODE_CAST_SHADOWS = 1 << 3
LIGHT_UNKNOWN, LIGHT_SPOT, LIGHT_POINT, LIGHT_DIRECTIONAL = 0, 1, 2, 3

# renderer/utils.rs:49-75, CubeMapFaceDescriptor::cube_faces(): (look, up) of +X, -X, +Y, -Y, +Z, -Z
CUBE_FACES = [((1, 0, 0), (0, -1, 0)), ((-1, 0, 0), (0, -1, 0)), ((0, 1, 0), (0, 0, 1)), ((0, -1, 0), (0, 0, -1)), ((0, 0, 1), (0, -1, 0)),
              ((0, 0, -1), (0, -1, 0))]


def dot3(u, v) -> np.float32:
    """nalgebra Vector3::dot, 3-element fast path: (a + b) + c (SURVEY Appendix A6)."""
    return (f32(u[0]) * f32(v[0]) + f32(u[1]) * f32(v[1])) + f32(u[2]) * f32(v[2])


def norm(v) -> np.float32:
    return np.sqrt(dot3(v, v))


def try_normalize(v, eps, fallback):
    """Vector3::try_normalize(eps).unwrap_or(fallback): norm <= eps ⇒ None."""
    n = norm(v)
    if n <= eps:
        return np.array(fallback, f32)
    return np.array([f32(v[0]) / n, f32(v[1]) / n, f32(v[2]) / n], f32)


def frustum_is_intersects_sphere(frustum: ob.Frustum, p, r) -> bool:
    """Frustum::is_intersects_sphere — fyrox-math/src/frustum.rs:336-347; Plane::dot = normal·p + d (plane.rs:78-80)."""
    r = f32(r)
    for pl in frustum.planes:
        d = dot3(pl.n, p) + f32(pl.d)
        if d < -r:
            return False
        if abs(d) < r:
            return True
    return True


def default_frustum() -> ob.Frustum:
    """Frustum::default — frustum.rs:32-43."""
    return ob.frustum_from_vp(ob.perspective(1.0, float(FRAC_PI_2), 0.01, 1024.0))


def shadow_maps(og: ob.Graph, flags, camera: ob.Frustum, camera_translation, render_mask, settings, sources, local_scale):
    """Every shadow map the reference renders for one camera, in its order, with its visible set.

    flags: the node flag words the graph was built with (cast_shadows = FYX_NODE_CAST_SHADOWS).
    settings: (spot_shadows_distance, point_shadows_distance, spot_shadows_enabled, point_shadows_enabled).
    sources: {node: (kind, full_cone_angle, distance_or_radius)}; local_scale: {node: (sx, sy, sz)} (missing = ones).
    Returns [(light, face, cascade, view_projection[16] f32, sorted visible node indices)].
    """
    spot_sd, point_sd, spot_en, point_en = f32(settings[0]), f32(settings[1]), bool(settings[2]), bool(settings[3])
    cam_t = np.asarray(camera_translation, f32)
    out = []
    # renderer/bundle.rs:926-974: light_sources = the camera's light list in pool order, Unknown kinds included
    for light in og.collect_lights(camera):
        light = int(light)
        if light not in sources:
            continue
        kind, full_cone_angle, raw = sources[light]
        if kind not in (LIGHT_SPOT, LIGHT_POINT):
            continue  # light.rs:560-568 Unknown: continue; Directional: cascaded shadow maps (shadow/csm.rs), not modelled
        g = og.global_transform(light)
        position = g[12:15].astype(f32)
        up_vector, look_vector = g[4:7].astype(f32), g[8:11].astype(f32)
        cast_shadows = bool(int(flags[light]) & NODE_CAST_SHADOWS)
        # light.rs:510
        distance_to_camera = norm(position - cam_t)
        # light.rs:512-559
        if kind == LIGHT_SPOT:
            shadows_distance = spot_sd
            shadows_enabled = cast_shadows and distance_to_camera <= spot_sd and spot_en
        else:
            shadows_distance = point_sd
            shadows_enabled = cast_shadows and distance_to_camera <= point_sd and point_en
        # light.rs:570-572
        scl = np.asarray(local_scale.get(light, (1.0, 1.0, 1.0)), f32)
        light_radius_scale = np.fmax(np.fmax(scl[0], scl[1]), scl[2])  # f32::max: a NaN operand yields the other
        light_radius = f32(light_radius_scale) * f32(raw)
        # light.rs:580-583
        emit_direction = try_normalize(up_vector, F32_EPSILON, (0.0, 0.0, 1.0))
        # light.rs:585-587
        if not frustum_is_intersects_sphere(camera, position, light_radius):
            continue
        # light.rs:589-602
        b1 = shadows_distance * f32(0.2)
        b2 = shadows_distance * f32(0.4)
        if distance_to_camera < b1 or norm(cam_t - position) <= light_radius:
            cascade = 0
        elif distance_to_camera > b1 and distance_to_camera < b2:
            cascade = 1
        else:
            cascade = 2
        # light.rs:651-684: use_light_occlusion_culling = false ⇒ needs_lighting stays true
        if not shadows_enabled:
            continue
        z_near, z_far = 0.01, float(light_radius)
        if kind == LIGHT_SPOT:
            # light.rs:697-722
            proj = ob.perspective(1.0, float(f32(full_cone_angle)), z_near, z_far)
            look_at = position - emit_direction
            up = try_normalize(look_vector, F32_EPSILON, (0.0, 1.0, 0.0))
            views = [(0, ob.look_at_rh(position, look_at, up))]
        else:
            # shadow/point.rs:166-180
            proj = ob.perspective(1.0, float(FRAC_PI_2), z_near, z_far)
            views = [(k, ob.look_at_rh(position, position + np.array(look, f32), np.array(up, f32))) for k, (look, up) in enumerate(CUBE_FACES)]
        for face, view in views:
            vp = ob.mat4_mul(proj, view)
            # shadow/spot.rs:142, shadow/point.rs:182: from_graph(.., render_mask, .., shadow pass); renderer/bundle.rs:893-896
            fr = ob.frustum_from_vp(vp) or default_frustum()
            vis = np.sort(og.from_graph(fr, render_mask, shadow_pass=True))
            out.append((light, face, cascade, vp, vis))
    return out

