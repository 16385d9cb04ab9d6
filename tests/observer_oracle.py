"""Oracle of fyx_cull_scene_observers: ObserversCollection::from_scene (renderer/observer.rs:88-153) with
Camera::calculate_matrices (scene/camera.rs:454-462), then one RenderDataBundleStorage::from_graph per observer
(renderer/mod.rs:1034-1047: frustum, LOD filter, static-batch Break, light list, environment map), in f32 numpy over the C
oracle's primitives (orc_look_at_rh, orc_mat4_mul, orc_frustum_from_view_projection_matrix, orc_from_graph_lod,
orc_collect_lights, orc_select_reflection_probe) and csm_oracle.projection_matrix for Projection::matrix.  Paths are
relative to the Fyrox tree.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

import csm_oracle as co
import oracle_binding as ob
import shadow_oracle as so

f32 = np.float32
NONE = 0xFFFFFFFF
PERSPECTIVE, ORTHOGRAPHIC = co.PERSPECTIVE, co.ORTHOGRAPHIC
ONCE, EACH_FRAME = 0, 1
PROBE_FACE, CAMERA = 0, 1
FOV_90 = f32(np.radians(f32(90.0)))  # 90f32.to_radians(): FRAC_PI_2 in f32


@dataclass
class Camera:
    """Camera::is_enabled, its Projection (fov in radians or vertical_size, z_near, z_far) and its render target's size
    ((0, 0) = none: the frame size of the call)."""
    projection: int = PERSPECTIVE
    fov_or_vertical_size: float = 1.2
    z_near: float = 0.1
    z_far: float = 200.0
    enabled: bool = True
    frame_size: tuple = (0.0, 0.0)


@dataclass
class Probe:
    """ReflectionProbe: update mode, z_near, z_far, rendering_position."""
    update_mode: int = ONCE
    z_near: float = 0.1
    z_far: float = 50.0
    rendering_position: tuple = (0.0, 0.0, 0.0)


class ProbeState:
    """ReflectionProbe::updated per probe node (probe.rs:166-173): True once rendered, cleared by a new record or
    force_update (probe.rs:215-218) and, for EachFrame probes, by every update (probe.rs:276-290)."""

    def __init__(self):
        self.rendered = {}

    def reset(self, nodes):
        for n in nodes:
            self.rendered[int(n)] = False


def projection(kind, fov_or_vertical_size, z_near, z_far, frame_size):
    """Projection::matrix(frame_size) (scene/camera.rs:89-174) through csm_oracle's restatement."""
    cam = co.CsmCamera(kind, float(f32(fov_or_vertical_size)), z_near, z_far, tuple(frame_size), np.eye(4, dtype=f32).reshape(16))
    return co.projection_matrix(cam, z_near, z_far)


def camera_matrices(g16, cam: Camera, frame_size):
    """Camera::calculate_matrices: look_at_rh(pos, pos + look, up) from the global matrix as it is, and the projection."""
    g = np.asarray(g16, f32)
    pos, up, look = g[12:15], g[4:7], g[8:11]
    view = ob.look_at_rh(pos, pos + look, up)
    fs = cam.frame_size if (cam.frame_size[0] != 0.0 or cam.frame_size[1] != 0.0) else frame_size
    return pos, view, projection(cam.projection, cam.fov_or_vertical_size, cam.z_near, cam.z_far, fs)


def probe_faces(g16, probe: Probe):
    """observer.rs:104-145: translation = global_rendering_position, one view per cube face, fov 90° and aspect 1."""
    t = np.asarray(g16, f32)[12:15] + np.asarray(probe.rendering_position, f32)
    proj = projection(PERSPECTIVE, FOV_90, probe.z_near, probe.z_far, (1.0, 1.0))
    return t, [(k, ob.look_at_rh(t, t + np.array(look, f32), np.array(up, f32)), proj) for k, (look, up) in enumerate(so.CUBE_FACES)]


def from_scene(og: ob.Graph, masks, cameras: dict, probes: dict, state: ProbeState, frame_size):
    """Every observer in the reference's order, with its visible set, light list and environment map.

    cameras / probes: {node: Camera / Probe}; masks: the nodes' render masks; state: the probes' rendered flags (updated
    as the reference's from_scene updates them).  Returns a list of dicts."""
    probe_obs, camera_obs = [], []
    lib = ob.lib()
    for node in sorted(set(cameras) | set(probes)):  # pool order
        if not lib.orc_node_is_alive(og.h, node) or not og.is_globally_enabled(node):  # observer.rs:91
            continue
        g = og.global_transform(node)
        if node in cameras:
            cam = cameras[node]
            if not cam.enabled:
                continue
            pos, view, proj = camera_matrices(g, cam, frame_size)
            camera_obs.append(dict(node=node, kind=CAMERA, face=0, translation=pos, z_near=f32(cam.z_near), z_far=f32(cam.z_far),
                                   view=view, projection=proj))
        elif node in probes:
            probe = probes[node]
            if probe.update_mode == ONCE and state.rendered.get(node, False):
                continue
            state.rendered[node] = True
            t, faces = probe_faces(g, probe)
            for k, view, proj in faces:
                probe_obs.append(dict(node=node, kind=PROBE_FACE, face=k, translation=t, z_near=f32(probe.z_near), z_far=f32(probe.z_far),
                                      view=view, projection=proj))
    out = probe_obs + camera_obs  # renderer/mod.rs:1364-1400: the probes first
    for o in out:
        o["render_mask"] = int(masks[o["node"]])
        o["view_projection"] = ob.mat4_mul(o["projection"], o["view"])
        fr = ob.frustum_from_vp(o["view_projection"]) or so.default_frustum()  # renderer/bundle.rs:893-896
        o["visible"] = np.sort(og.from_graph_lod(fr, o["translation"], o["z_near"], o["z_far"], o["render_mask"]))
        o["lights"] = og.collect_lights(fr)
        t = np.ascontiguousarray(o["translation"], f32)
        o["environment_map"] = int(lib.orc_select_reflection_probe(og.h, ob.fp(t))) if o["kind"] == CAMERA else NONE
    return out
