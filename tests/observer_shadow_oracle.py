"""Oracle of fyx_cull_scene_shadow_casters: the deferred light renderer's shadow loop (renderer/light.rs:509-782) for every
observer of render_scene_observer (renderer/mod.rs:964-1120), over observer_oracle.from_scene and csm_oracle.shadow_maps.
Each observer is the camera of its own loop: its frustum, translation and render mask, and a CsmCamera built from it.  Each
map's list is from_graph with the map's own LOD observer and static-batch Break (og.from_graph_lod, as
tests/test_gpu_shadow_pruned.py checks fyx_cull_shadow_casters_pruned).  Paths are relative to the Fyrox tree.
"""
from __future__ import annotations

import numpy as np

import csm_oracle as co
import observer_oracle as oo
import oracle_binding as ob
import shadow_oracle as so

f32 = np.float32


def csm_camera(o, cameras, frame_size, csm_enabled=True, options=None, probe_frame=(1.0, 1.0)):
    """The CsmCamera of observer `o` (a row of observer_oracle.from_scene): a camera's projection, raw z range, view and
    frame size (its render target's when not 0,0, else the call's); a probe face's fov 90° and a square frame
    (`probe_frame`: any square size gives the same matrices, Projection::matrix uses only w / h)."""
    options = {} if options is None else options
    if o["kind"] == oo.CAMERA:
        cam = cameras[o["node"]]
        fs = cam.frame_size if (cam.frame_size[0] != 0.0 or cam.frame_size[1] != 0.0) else frame_size
        return co.CsmCamera(cam.projection, cam.fov_or_vertical_size, cam.z_near, cam.z_far, tuple(fs), o["view"], bool(csm_enabled), dict(options))
    return co.CsmCamera(oo.PERSPECTIVE, oo.FOV_90, float(o["z_near"]), float(o["z_far"]), tuple(probe_frame), o["view"], bool(csm_enabled),
                        dict(options))


def map_observer(og, light, cascade, sources, local_scale, csm: co.CsmCamera):
    """(translation, z_near, z_far) of a map's from_graph: the light's position, 0.01 and the radius for spot and point maps
    (light.rs:700-728, shadow/point.rs:162-190); the look_at_lh eye and the slice's depths for cascade i (csm.rs:195-270)."""
    g = og.global_transform(light)
    if sources[light][0] == so.LIGHT_DIRECTIONAL:
        with np.errstate(all="ignore"):
            zn, zf = co.cascade_depths(csm, csm.options.get(light, co.CSM_DEFAULT), cascade)
            light_direction = -so.try_normalize(g[4:7].astype(f32), so.F32_EPSILON, (0.0, 1.0, 0.0))
            center = co.frustum_center(co.slice_corners(csm, zn, zf))
            return center + light_direction, f32(zn), f32(zf)
    scl = np.asarray(local_scale.get(light, (1.0, 1.0, 1.0)), f32)
    radius = f32(np.fmax(np.fmax(scl[0], scl[1]), scl[2])) * f32(sources[light][2])
    return g[12:15].astype(f32), f32(0.01), radius


def observer_maps(og, flags, o, cameras, frame_size, settings, sources, local_scale, csm_enabled=True, options=None, probe_frame=(1.0, 1.0)):
    """The maps observer `o` renders, in its loop's order: [dict(light, face, cascade, view_projection, observer, mask,
    visible)]."""
    fr = ob.frustum_from_vp(o["view_projection"]) or so.default_frustum()
    cam = csm_camera(o, cameras, frame_size, csm_enabled, options, probe_frame)
    mask = int(o["render_mask"])
    out = []
    for light, face, cascade, vp, _ in co.shadow_maps(og, flags, fr, o["translation"], mask, settings, sources, local_scale, csm=cam):
        t, zn, zf = map_observer(og, light, cascade, sources, local_scale, cam)
        mfr = ob.frustum_from_vp(vp) or so.default_frustum()
        vis = np.sort(og.from_graph_lod(mfr, t, zn, zf, mask, shadow_pass=True))
        out.append(dict(light=light, face=face, cascade=cascade, view_projection=vp, observer=(t, zn, zf), mask=mask, visible=vis))
    return out


def scene_shadow_maps(og, flags, observers, cameras, frame_size, settings, sources, local_scale, csm_enabled=True, options=None):
    """Per observer of `observers` (observer_oracle.from_scene's list, in its order), its ordered maps."""
    return [observer_maps(og, flags, o, cameras, frame_size, settings, sources, local_scale, csm_enabled, options) for o in observers]
