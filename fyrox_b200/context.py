"""Thin numpy-facing wrapper over the C ABI (one method per ``fyx_*`` entry point).

All compute happens in libfyrox_b200.so's sm_90a kernels; this file only marshals arguments.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import numpy as np

from . import _lib as L


class FyxError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"fyx error {code}: {msg}")
        self.code = code


def _u32(a) -> Optional[np.ndarray]:
    if a is None:
        return None
    return np.ascontiguousarray(a, dtype=np.uint32)


def _f32(a) -> Optional[np.ndarray]:
    if a is None:
        return None
    return np.ascontiguousarray(a, dtype=np.float32)


def _ptr(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


ANIMATED_VERTEX_LAYOUT = L.fyx_vertex_layout(68, 0, 20, 48, 64)  # scene/mesh/vertex.rs:140-210


def frustum_from_view_projection_matrix(vp) -> Optional[L.fyx_frustum]:
    """Frustum::from_view_projection_matrix (fyrox-math/src/frustum.rs:54-82); None where the reference returns None."""
    lib = L.load()
    m = _f32(np.asarray(vp, dtype=np.float32).reshape(-1))
    assert m.size == 16
    f = L.fyx_frustum()
    rc = lib.fyx_frustum_from_view_projection_matrix(m.ctypes.data_as(L.f32p), C.byref(f))
    return f if rc == 0 else None


def frustum_default() -> L.fyx_frustum:
    f = L.fyx_frustum()
    L.load().fyx_frustum_default(C.byref(f))
    return f


def mat4_mul(a, b) -> np.ndarray:
    """Matrix4 * Matrix4 in nalgebra's order, on 16-float column-major arrays."""
    a = _f32(np.asarray(a).reshape(-1))
    b = _f32(np.asarray(b).reshape(-1))
    out = np.empty(16, dtype=np.float32)
    L.load().fyx_mat4_mul(a.ctypes.data_as(L.f32p), b.ctypes.data_as(L.f32p), out.ctypes.data_as(L.f32p))
    return out


def frustum_to_numpy(f: L.fyx_frustum):
    planes = np.array([[f.planes[p][k] for k in range(4)] for p in range(6)], dtype=np.float32)
    corners = np.array([[f.corners[i][k] for k in range(3)] for i in range(8)], dtype=np.float32)
    return planes, corners


def frustum_from_numpy(planes, corners) -> L.fyx_frustum:
    f = L.fyx_frustum()
    for p in range(6):
        for k in range(4):
            f.planes[p][k] = float(planes[p][k])
    for i in range(8):
        for k in range(3):
            f.corners[i][k] = float(corners[i][k])
    return f


class PinnedBuffer:
    """Page-locked host memory from fyx_host_alloc, viewed as a numpy array."""

    def __init__(self, shape, dtype):
        self._lib = L.load()
        self.dtype = np.dtype(dtype)
        self.shape = tuple(int(s) for s in (shape if isinstance(shape, (tuple, list)) else (shape,)))
        nbytes = int(np.prod(self.shape)) * self.dtype.itemsize
        self.ptr = self._lib.fyx_host_alloc(max(nbytes, 1))
        if not self.ptr:
            raise MemoryError("fyx_host_alloc failed")
        buf = (C.c_char * max(nbytes, 1)).from_address(self.ptr)
        self.array = np.frombuffer(buf, dtype=self.dtype, count=int(np.prod(self.shape))).reshape(self.shape)

    def free(self):
        if self.ptr:
            self.array = None
            self._lib.fyx_host_free(self.ptr)
            self.ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class Context:
    """One fyx_ctx (one GPU)."""

    def __init__(self, device: int = -1, stream: Optional[int] = None):
        self._lib = L.load()
        cfg = L.fyx_config(C.sizeof(L.fyx_config), device, stream, 0)
        h = L.ctx_p()
        rc = self._lib.fyx_create(C.byref(cfg), C.byref(h))
        if rc != 0:
            raise FyxError(rc, (self._lib.fyx_last_error(None) or b"").decode())
        self._h = h
        self.n_nodes = 0
        self._surfaces = []  # (n_bones, n_verts)

    # -- plumbing --
    def _chk(self, rc: int):
        if rc != 0:
            raise FyxError(rc, (self._lib.fyx_last_error(self._h) or b"").decode())

    def close(self):
        if getattr(self, "_h", None):
            self._lib.fyx_destroy(self._h)
            self._h = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def handle(self):
        return self._h

    def sync(self):
        self._chk(self._lib.fyx_sync(self._h))

    # -- scene description --
    def set_topology(self, parent, flags=None, render_mask=None, local_aabb=None, root: int = 0, global_index=None):
        parent = _u32(parent)
        n = parent.size
        flags, render_mask, global_index = _u32(flags), _u32(render_mask), _u32(global_index)
        local_aabb = _f32(local_aabb)
        for a, k in ((flags, 1), (render_mask, 1), (global_index, 1), (local_aabb, 6)):
            assert a is None or a.size == n * k
        self._chk(self._lib.fyx_set_topology(self._h, n, root, _ptr(parent), _ptr(flags), _ptr(render_mask), _ptr(local_aabb), _ptr(global_index)))
        self.n_nodes = n

    def set_dfs_order(self, preorder_rank):
        """Pre-order DFS rank of every node (children order of the host graph); None clears it."""
        r = _u32(preorder_rank)
        self._chk(self._lib.fyx_set_dfs_order(self._h, 0 if r is None else r.size, _ptr(r)))

    def set_local_matrices(self, m16, idx=None):
        m16 = _f32(m16)
        idx = _u32(idx)
        count = m16.size // 16
        assert idx is None or idx.size == count
        self._chk(self._lib.fyx_set_local_matrices(self._h, count, _ptr(idx), _ptr(m16)))

    def set_local_trs(self, trs, idx=None):
        """trs: (count, 10) f32 rows of position xyz, rotation quaternion ijkw, scale xyz (fyx_trs)."""
        trs = _f32(trs)
        idx = _u32(idx)
        count = trs.size // 10
        assert idx is None or idx.size == count
        self._chk(self._lib.fyx_set_local_trs(self._h, count, _ptr(idx), _ptr(trs)))

    def set_local_rotations(self, quats, idx=None):
        """quats: (count, 4) f32 unit quaternions i,j,k,w; position/scale stay what the last set_local_trs sent."""
        q = _f32(quats)
        idx = _u32(idx)
        count = q.size // 4
        assert idx is None or idx.size == count
        self._chk(self._lib.fyx_set_local_rotations(self._h, count, _ptr(idx), _ptr(q)))

    def set_transform_statics(self, statics, idx=None):
        """statics: (count, 25) f32 rows: pre_rotation ijkw, post_rotation_matrix (9, column-major), rotation_offset,
        rotation_pivot, scaling_offset, scaling_pivot (fyx_transform_statics)."""
        statics = _f32(statics)
        idx = _u32(idx)
        count = statics.size // 25
        assert idx is None or idx.size == count
        self._chk(self._lib.fyx_set_transform_statics(self._h, count, _ptr(idx), _ptr(statics)))

    def set_flags(self, flags, idx=None):
        flags, idx = _u32(flags), _u32(idx)
        self._chk(self._lib.fyx_set_flags(self._h, flags.size, _ptr(idx), _ptr(flags)))

    def set_render_masks(self, masks, idx=None):
        masks, idx = _u32(masks), _u32(idx)
        self._chk(self._lib.fyx_set_render_masks(self._h, masks.size, _ptr(idx), _ptr(masks)))

    def set_local_aabbs(self, aabbs, idx=None):
        aabbs, idx = _f32(aabbs), _u32(idx)
        self._chk(self._lib.fyx_set_local_aabbs(self._h, aabbs.size // 6, _ptr(idx), _ptr(aabbs)))

    def add_skinned_surface(self, mesh_node: int, bone_nodes, inv_bind_m16, verts=None, layout: L.fyx_vertex_layout = None, n_verts: int = None) -> int:
        bone_nodes = _u32(bone_nodes)
        inv_bind = _f32(inv_bind_m16)
        assert inv_bind.size == bone_nodes.size * 16
        if verts is None:
            n_verts, vptr, lay = 0, None, None
        else:
            lay = layout or ANIMATED_VERTEX_LAYOUT
            if isinstance(verts, np.ndarray):
                verts = np.ascontiguousarray(verts)
                if n_verts is None:
                    n_verts = verts.nbytes // lay.stride
                vptr = verts.ctypes.data_as(C.c_void_p)
            else:  # raw address
                vptr = C.c_void_p(int(verts))
                assert n_verts is not None
        sid = C.c_uint32()
        self._chk(
            self._lib.fyx_add_skinned_surface(
                self._h, mesh_node, bone_nodes.size, _ptr(bone_nodes), _ptr(inv_bind), n_verts, vptr, C.byref(lay) if lay is not None else None, C.byref(sid)
            )
        )
        self._surfaces.append((int(bone_nodes.size), int(n_verts)))
        return sid.value

    def set_blend_shapes(self, surface_id: int, records, weights=None):
        """BlendShapesContainer of a surface: records = uint16 array (n_shapes, layer_stride, 9) of binary16 bit patterns
        (position, normal, tangent offsets per vertex, scene/mesh/surface.rs:92-218); weights = BlendShape::weight (0..100)."""
        r = np.ascontiguousarray(records, dtype=np.uint16)
        if r.size == 0:
            self._chk(self._lib.fyx_set_blend_shapes(self._h, surface_id, 0, None, 0, None))
            return
        assert r.ndim == 3 and r.shape[2] == 9
        w = None if weights is None else np.ascontiguousarray(weights, dtype=np.float32)
        assert w is None or w.size == r.shape[0]
        self._chk(self._lib.fyx_set_blend_shapes(self._h, surface_id, r.shape[0], r.ctypes.data_as(C.c_void_p), r.shape[1], _ptr(w)))

    def set_blend_shape_weights(self, surface_id: int, weights):
        w = np.ascontiguousarray(weights, dtype=np.float32)
        self._chk(self._lib.fyx_set_blend_shape_weights(self._h, surface_id, w.size, _ptr(w)))

    def reserve_skinning(self, total_bones: int, total_verts: int):
        self._chk(self._lib.fyx_reserve_skinning(self._h, total_bones, total_verts))

    def commit_surfaces(self):
        self._chk(self._lib.fyx_commit_surfaces(self._h))

    # -- per frame --
    def update_transforms(self, flags: int = L.UPDATE_INCREMENTAL):
        self._chk(self._lib.fyx_update_transforms(self._h, flags))

    @staticmethod
    def _frusta(frusta: Sequence[L.fyx_frustum]):
        arr = (L.fyx_frustum * max(len(frusta), 1))()
        for i, f in enumerate(frusta):
            arr[i] = f
        return arr

    def cull(self, frusta, cam_mask=None, pass_flags=None):
        arr = self._frusta(frusta)
        cm, pf = _u32(cam_mask), _u32(pass_flags)
        self._chk(self._lib.fyx_cull(self._h, len(frusta), arr, _ptr(cm), _ptr(pf)))

    def update_and_cull(self, frusta, update_flags: int = L.UPDATE_INCREMENTAL, cam_mask=None, pass_flags=None):
        arr = self._frusta(frusta)
        cm, pf = _u32(cam_mask), _u32(pass_flags)
        self._chk(self._lib.fyx_update_and_cull(self._h, update_flags, len(frusta), arr, _ptr(cm), _ptr(pf)))

    def get_visible(self, frustum: int = 0, copy: bool = True) -> np.ndarray:
        """Visible node indices of one frustum.  copy=False returns a view of the library's pinned buffer
        (valid until the next cull / frame on this context)."""
        p = L.u32p()
        n = C.c_uint32()
        self._chk(self._lib.fyx_get_visible(self._h, frustum, C.byref(p), C.byref(n)))
        if n.value == 0:
            return np.empty(0, dtype=np.uint32)
        v = np.ctypeslib.as_array(p, shape=(n.value,))
        return v.copy() if copy else v

    def get_visible_device(self, frustum: int = 0):
        d_idx, d_cnt = C.c_void_p(), C.c_void_p()
        self._chk(self._lib.fyx_get_visible_device(self._h, frustum, C.byref(d_idx), C.byref(d_cnt)))
        return d_idx.value, d_cnt.value

    # ---- N4 (LOD filter) ----
    def set_lod_ranges(self, begin_end, idx=None):
        """Per LOD object the [begin, end] of its level (renderer/bundle.rs:898-916); begin NaN removes the node."""
        be = _f32(begin_end)
        ix = _u32(idx)
        self._chk(self._lib.fyx_set_lod_ranges(self._h, be.size // 2, _ptr(ix), _ptr(be)))

    def set_observers(self, observers):
        """observers = [(translation xyz, z_near, z_far), ...], one per frustum of the culls that follow; [] switches LOD off."""
        arr = (L.fyx_observer * max(len(observers), 1))()
        for k, (t, zn, zf) in enumerate(observers):
            arr[k].translation[:] = [float(x) for x in t]
            arr[k].z_near, arr[k].z_far = float(zn), float(zf)
        self._chk(self._lib.fyx_set_observers(self._h, len(observers), C.cast(arr, C.c_void_p)))
        self._n_observers = len(observers)

    # ---- N4 (light list) ----
    def cull_lights(self):
        """Light sources seen by every frustum of the most recent cull (renderer/bundle.rs:926-974)."""
        self._chk(self._lib.fyx_cull_lights(self._h))

    def select_reflection_probes(self) -> np.ndarray:
        """Per observer (set_observers): the reflection probe from_graph would pick (renderer/bundle.rs:918-925), FYX_NONE = none."""
        n = getattr(self, "_n_observers", 0)
        out = np.full(max(n, 1), L.FYX_NONE, np.uint32)
        self._chk(self._lib.fyx_select_reflection_probes(self._h, n, out.ctypes.data_as(C.c_void_p)))
        return out[:n]

    def get_visible_lights(self, frustum: int = 0) -> np.ndarray:
        p = L.u32p()
        n = C.c_uint32()
        self._chk(self._lib.fyx_get_visible_lights(self._h, frustum, C.byref(p), C.byref(n)))
        if n.value == 0:
            return np.empty(0, dtype=np.uint32)
        return np.ctypeslib.as_array(p, shape=(n.value,)).copy()

    # ---- N4 (shadow casters) ----
    LIGHT_SOURCE_DTYPE = np.dtype([("kind", "<u4"), ("full_cone_angle", "<f4"), ("distance_or_radius", "<f4")])
    SHADOW_MAP_DTYPE = np.dtype([("light", "<u4"), ("face", "<u4"), ("cascade", "<u4"), ("first", "<u4"), ("count", "<u4"),
                                 ("view_projection", "<f4", 16)])

    def set_light_sources(self, sources, idx=None):
        """One record per light node (LIGHT_SOURCE_DTYPE: kind, full_cone_angle, distance_or_radius); kind LIGHT_UNKNOWN removes it."""
        src = np.ascontiguousarray(sources, dtype=self.LIGHT_SOURCE_DTYPE)
        ix = _u32(idx)
        self._chk(self._lib.fyx_set_light_sources(self._h, src.size, _ptr(ix), src.ctypes.data_as(C.c_void_p)))

    CSM_OPTIONS_DTYPE = np.dtype([("relative", "<u4"), ("splits", "<f4", 3)])

    def set_csm_options(self, options, idx=None):
        """FrustumSplitOptions per directional light node (CSM_OPTIONS_DTYPE: relative 0 = Absolute far planes, 1 = Relative
        fractions; splits).  Nodes without a record use Absolute {5, 25, 64}."""
        opt = np.ascontiguousarray(options, dtype=self.CSM_OPTIONS_DTYPE)
        ix = _u32(idx)
        self._chk(self._lib.fyx_set_csm_options(self._h, opt.size, _ptr(ix), opt.ctypes.data_as(C.c_void_p)))

    @staticmethod
    def csm_camera(view_matrix, frame_size, z_near: float, z_far: float, fov: float | None = None, vertical_size: float | None = None,
                   csm_enabled: bool = True):
        """The camera of the cascaded shadow maps: a perspective projection (fov in radians) or an orthographic one
        (vertical_size), its own z_near / z_far, Camera::view_matrix and the frame size the cascades are rendered for."""
        if (fov is None) == (vertical_size is None):
            raise ValueError("give exactly one of fov (perspective) and vertical_size (orthographic)")
        cam = L.fyx_csm_camera()
        cam.projection = L.PROJECTION_PERSPECTIVE if fov is not None else L.PROJECTION_ORTHOGRAPHIC
        cam.fov_or_vertical_size = float(fov if fov is not None else vertical_size)
        cam.z_near, cam.z_far = float(z_near), float(z_far)
        cam.frame_size[:] = [float(v) for v in frame_size]
        cam.view_matrix[:] = [float(v) for v in np.asarray(view_matrix, np.float32).reshape(16)]
        cam.csm_enabled = int(bool(csm_enabled))
        return cam

    def cull_shadow_casters(self, camera_frustum: int, camera_translation, spot_shadows_distance: float = 10.0, point_shadows_distance: float = 10.0,
                            spot_shadows_enabled: bool = True, point_shadows_enabled: bool = True, csm_camera=None, prune: bool = False):
        """The shadow maps the deferred light renderer draws for frustum `camera_frustum` of the last cull, and their visible
        sets (renderer/light.rs:509-606, 695-782).  Defaults are QualitySettings::default() (renderer/settings.rs).  Spot and
        point maps always; the cascades of directional lights (renderer/shadow/csm.rs) when `csm_camera` (Context.csm_camera
        or an fyx_csm_camera) is given, through fyx_cull_shadow_casters_csm.  prune=True: every map's list with the map's own
        LOD filter and static-batch pruning (fyx_cull_shadow_casters_pruned, with or without `csm_camera`); without it a scene
        with LOD ranges or static batches is refused."""
        t = _f32(camera_translation)
        st = L.fyx_shadow_settings(float(spot_shadows_distance), float(point_shadows_distance), int(bool(spot_shadows_enabled)),
                                   int(bool(point_shadows_enabled)))
        if prune:
            cam = C.byref(csm_camera) if csm_camera is not None else None
            self._chk(self._lib.fyx_cull_shadow_casters_pruned(self._h, camera_frustum, t.ctypes.data_as(L.f32p), C.byref(st), cam))
        elif csm_camera is None:
            self._chk(self._lib.fyx_cull_shadow_casters(self._h, camera_frustum, t.ctypes.data_as(L.f32p), C.byref(st)))
        else:
            self._chk(self._lib.fyx_cull_shadow_casters_csm(self._h, camera_frustum, t.ctypes.data_as(L.f32p), C.byref(st), C.byref(csm_camera)))

    def get_shadow_maps(self, copy: bool = True):
        """(maps, entries): maps is a SHADOW_MAP_DTYPE array; map k's visible set is entries[first:first + count].
        copy=False returns views of the library's pinned buffers, valid until the next cull_shadow_casters."""
        pm, pe = C.c_void_p(), C.c_void_p()
        n = C.c_uint32()
        self._chk(self._lib.fyx_get_shadow_maps(self._h, C.byref(pm), C.byref(n), C.byref(pe)))
        if not n.value:
            return np.empty(0, self.SHADOW_MAP_DTYPE), np.empty(0, np.uint32)
        maps = np.frombuffer((C.c_char * (n.value * self.SHADOW_MAP_DTYPE.itemsize)).from_address(pm.value), self.SHADOW_MAP_DTYPE)
        total = int(maps["first"][-1]) + int(maps["count"][-1])
        entries = np.ctypeslib.as_array(C.cast(pe.value, L.u32p), shape=(max(total, 1),))[:total]
        return (maps.copy(), entries.copy()) if copy else (maps, entries)

    def get_shadow_maps_device(self):
        """(device pointer of the map table, number of maps, device pointer of the entries)."""
        pm, pe = C.c_void_p(), C.c_void_p()
        n = C.c_uint32()
        self._chk(self._lib.fyx_get_shadow_maps_device(self._h, C.byref(pm), C.byref(n), C.byref(pe)))
        return pm.value, n.value, pe.value

    # ---- N4 (scene observers) ----
    CAMERA_DTYPE = np.dtype([("enabled", "<u4"), ("projection", "<u4"), ("fov_or_vertical_size", "<f4"), ("z_near", "<f4"), ("z_far", "<f4"),
                             ("frame_size", "<f4", 2)])
    PROBE_DTYPE = np.dtype([("present", "<u4"), ("update_mode", "<u4"), ("z_near", "<f4"), ("z_far", "<f4"), ("rendering_position", "<f4", 3)])
    SCENE_OBSERVER_DTYPE = np.dtype([(n, "<u4") for n in ("node", "kind", "face", "render_mask", "first", "count", "lights_first", "lights_count",
                                                          "environment_map")]
                                    + [("translation", "<f4", 3), ("z_near", "<f4"), ("z_far", "<f4"), ("view", "<f4", 16),
                                       ("projection", "<f4", 16), ("view_projection", "<f4", 16)])

    def set_cameras(self, idx, cameras):
        """Camera records (CAMERA_DTYPE) of the nodes `idx`; projection PROJECTION_NONE removes a node's record."""
        idx = _u32(idx)
        recs = np.ascontiguousarray(cameras, self.CAMERA_DTYPE)
        self._chk(self._lib.fyx_set_cameras(self._h, recs.size, _ptr(idx), recs.ctypes.data))

    def set_reflection_probes(self, idx, probes):
        """Reflection-probe records (PROBE_DTYPE) of the nodes `idx`; present 0 removes a node's record."""
        idx = _u32(idx)
        recs = np.ascontiguousarray(probes, self.PROBE_DTYPE)
        self._chk(self._lib.fyx_set_reflection_probes(self._h, recs.size, _ptr(idx), recs.ctypes.data))

    def force_reflection_probe_update(self, idx):
        idx = _u32(idx)
        self._chk(self._lib.fyx_force_reflection_probe_update(self._h, idx.size, _ptr(idx)))

    def cull_scene_observers(self, frame_size):
        """ObserversCollection::from_scene and one from_graph per observer (fyx_cull_scene_observers)."""
        fs = np.ascontiguousarray(frame_size, np.float32).reshape(2)
        self._chk(self._lib.fyx_cull_scene_observers(self._h, fs.ctypes.data_as(L.f32p)))

    def get_scene_observers(self):
        """(table, entries, light_entries): table is a SCENE_OBSERVER_DTYPE array; observer o's visible set is
        entries[first:first + count], its lights light_entries[lights_first:lights_first + lights_count]."""
        pt, pe, pl = C.c_void_p(), C.c_void_p(), C.c_void_p()
        n = C.c_uint32()
        self._chk(self._lib.fyx_get_scene_observers(self._h, C.byref(pt), C.byref(n), C.byref(pe), C.byref(pl)))
        if not n.value:
            return np.empty(0, self.SCENE_OBSERVER_DTYPE), np.empty(0, np.uint32), np.empty(0, np.uint32)
        table = np.frombuffer((C.c_char * (n.value * self.SCENE_OBSERVER_DTYPE.itemsize)).from_address(pt.value), self.SCENE_OBSERVER_DTYPE).copy()
        total = int(table["first"][-1]) + int(table["count"][-1])
        ltotal = int(table["lights_first"][-1]) + int(table["lights_count"][-1])
        entries = np.ctypeslib.as_array(C.cast(pe.value, L.u32p), shape=(max(total, 1),))[:total].copy()
        lights = np.ctypeslib.as_array(C.cast(pl.value, L.u32p), shape=(max(ltotal, 1),))[:ltotal].copy()
        return table, entries, lights

    def get_scene_observers_device(self):
        """(device pointer of the table, number of observers, device pointers of the entries and light entries)."""
        pt, pe, pl = C.c_void_p(), C.c_void_p(), C.c_void_p()
        n = C.c_uint32()
        self._chk(self._lib.fyx_get_scene_observers_device(self._h, C.byref(pt), C.byref(n), C.byref(pe), C.byref(pl)))
        return pt.value, n.value, pe.value, pl.value

    SCENE_SHADOW_MAP_DTYPE = np.dtype([("observer", "<u4"), ("map", "<u4")])

    def cull_scene_shadow_casters(self, spot_shadows_distance: float = 10.0, point_shadows_distance: float = 10.0, spot_shadows_enabled: bool = True,
                                  point_shadows_enabled: bool = True, csm_enabled: bool = True):
        """The shadow maps every observer of the last cull_scene_observers renders (fyx_cull_scene_shadow_casters): the map
        table and lists of get_shadow_maps, spot and point maps shared between observers, and the refs of
        get_scene_shadow_maps.  Defaults are QualitySettings::default() (renderer/settings.rs)."""
        st = L.fyx_shadow_settings(float(spot_shadows_distance), float(point_shadows_distance), int(bool(spot_shadows_enabled)),
                                   int(bool(point_shadows_enabled)))
        self._chk(self._lib.fyx_cull_scene_shadow_casters(self._h, C.byref(st), int(bool(csm_enabled))))

    def get_scene_shadow_maps(self) -> np.ndarray:
        """SCENE_SHADOW_MAP_DTYPE refs (observer, map) in render order: `map` is a row of get_shadow_maps' table."""
        p = C.c_void_p()
        n = C.c_uint32()
        self._chk(self._lib.fyx_get_scene_shadow_maps(self._h, C.byref(p), C.byref(n)))
        if not n.value:
            return np.empty(0, self.SCENE_SHADOW_MAP_DTYPE)
        return np.frombuffer((C.c_char * (n.value * self.SCENE_SHADOW_MAP_DTYPE.itemsize)).from_address(p.value), self.SCENE_SHADOW_MAP_DTYPE).copy()

    def get_scene_shadow_maps_device(self):
        """(device pointer of the refs, number of refs)."""
        p = C.c_void_p()
        n = C.c_uint32()
        self._chk(self._lib.fyx_get_scene_shadow_maps_device(self._h, C.byref(p), C.byref(n)))
        return p.value, n.value

    def pack_scene_observer_instances(self):
        """Pack the instances of every observer of the last cull_scene_observers (made with enable_instances) in one call."""
        self._chk(self._lib.fyx_pack_scene_observer_instances(self._h))

    def get_scene_observer_instances(self, observer: int) -> dict:
        """Instances of observer `observer`: the same dict as pack_instances, for its view and view_projection."""
        out = L.fyx_instances()
        self._chk(self._lib.fyx_get_scene_observer_instances(self._h, observer, C.byref(out)))
        return self._instances_dict(out, self._instance_surfaces(self._lib.fyx_get_scene_observer_instance_surfaces, observer, out.count))

    def pack_scene_observer_bone_matrices(self):
        self._chk(self._lib.fyx_pack_scene_observer_bone_matrices(self._h))

    def get_scene_observer_bone_matrix_block(self, observer: int, instance: int):
        """(255,16) f32 block of instance `instance` of observer `observer`, or None for an unskinned instance."""
        return self._bone_matrix_block(self._lib.fyx_get_scene_observer_bone_matrix_block, observer, instance)

    # ---- N2: animation sampling on the device ----
    KEY_DTYPE = np.dtype([("location", "<f4"), ("value", "<f4"), ("kind", "<u4"), ("left_tangent", "<f4"), ("right_tangent", "<f4")])
    TRACK_DTYPE = np.dtype([("target_node", "<u4"), ("binding", "<u4"), ("value_kind", "<u4"), ("enabled", "<u4"), ("n_curves", "<u4"),
                            ("first_key", "<u4", 4), ("n_keys", "<u4", 4)])

    def anim_add(self, tracks, keys, speed=1.0, looped=True, time_slice=(0.0, 0.0), time_position=0.0, enabled=True) -> int:
        """Add an Animation (fyrox-animation/src/lib.rs): tracks = TRACK_DTYPE array, keys = KEY_DTYPE array."""
        tracks = np.ascontiguousarray(tracks, dtype=self.TRACK_DTYPE)
        keys = np.ascontiguousarray(keys, dtype=self.KEY_DTYPE)
        d = L.fyx_animation_desc()
        d.struct_size = C.sizeof(L.fyx_animation_desc)
        d.n_tracks, d.tracks = len(tracks), tracks.ctypes.data
        d.n_keys, d.keys = len(keys), keys.ctypes.data
        d.speed, d.time_position = float(speed), float(time_position)
        d.time_slice_start, d.time_slice_end = float(time_slice[0]), float(time_slice[1])
        d.looped, d.enabled = int(bool(looped)), int(bool(enabled))
        out = C.c_uint32()
        self._chk(self._lib.fyx_anim_add(self._h, C.byref(d), C.byref(out)))
        return out.value

    def anim_clear(self):
        self._chk(self._lib.fyx_anim_clear(self._h))

    def anim_set_enabled(self, anim: int, enabled: bool):
        self._chk(self._lib.fyx_anim_set_enabled(self._h, anim, int(bool(enabled))))

    def anim_set_track_enabled(self, anim: int, track: int, enabled: bool):
        self._chk(self._lib.fyx_anim_set_track_enabled(self._h, anim, track, int(bool(enabled))))

    def anim_set_speed(self, anim: int, speed: float):
        self._chk(self._lib.fyx_anim_set_speed(self._h, anim, float(speed)))

    def anim_set_time_position(self, anim: int, t: float):
        self._chk(self._lib.fyx_anim_set_time_position(self._h, anim, float(t)))

    def anim_time_positions(self, first: int, count: int) -> np.ndarray:
        """Animation::time_position() of `count` animations starting at `first` (read back from the device)."""
        out = np.empty(count, dtype=np.float32)
        self._chk(self._lib.fyx_anim_get_time_positions(self._h, first, count, out.ctypes.data_as(C.c_void_p)))
        return out

    def anim_blend_group(self, anims, weights) -> int:
        """BlendAnimations over PlayAnimation sources with constant weights (machine/node/blend.rs:136-166)."""
        a = np.ascontiguousarray(anims, dtype=np.uint32)
        w = np.ascontiguousarray(weights, dtype=np.float32)
        assert a.size == w.size
        out = C.c_uint32()
        self._chk(self._lib.fyx_anim_blend_group(self._h, a.size, _ptr(a), _ptr(w), C.byref(out)))
        return out.value

    def anim_set_blend_weights(self, group: int, weights):
        w = np.ascontiguousarray(weights, dtype=np.float32)
        self._chk(self._lib.fyx_anim_set_blend_weights(self._h, group, w.size, _ptr(w)))

    def animate(self, dt: float):
        """AnimationContainer::update_animations(dt) for every animation (scene/animation/mod.rs:83-88)."""
        self._chk(self._lib.fyx_animate(self._h, float(dt)))

    SIGNAL_DTYPE = np.dtype([("time", "<f4"), ("enabled", "<u4")])
    EVENT_DTYPE = np.dtype([("anim", "<u4"), ("signal", "<u4")])
    ROOT_MOTION_DTYPE = np.dtype([("delta_position", "<f4", 3), ("delta_rotation", "<f4", 4), ("present", "<u4")])

    def anim_set_signals(self, anim: int, signals):
        """Replace animation `anim`'s signals: a sequence of (time, enabled) or a SIGNAL_DTYPE array.  Events name a
        signal by its index in this list."""
        s = np.array([tuple(x) for x in signals], self.SIGNAL_DTYPE) if not isinstance(signals, np.ndarray) else signals
        s = np.ascontiguousarray(s, dtype=self.SIGNAL_DTYPE)
        self._chk(self._lib.fyx_anim_set_signals(self._h, anim, len(s), s.ctypes.data_as(C.c_void_p) if len(s) else None))

    def anim_set_signal_enabled(self, anim: int, signal: int, enabled: bool):
        self._chk(self._lib.fyx_anim_set_signal_enabled(self._h, anim, signal, int(bool(enabled))))

    def anim_set_max_event_capacity(self, anim: int, capacity: int):
        self._chk(self._lib.fyx_anim_set_max_event_capacity(self._h, anim, int(capacity)))

    def anim_take_events(self, max_events: Optional[int] = None):
        """(EVENT_DTYPE array, lost): Animation::take_events of every animation, grouped by animation in ascending order;
        `lost` counts the events dropped because a store was full since the last call.  max_events None = every queued
        event; otherwise the rest stays queued."""
        chunk = 4096 if max_events is None else int(max_events)
        parts, lost_total = [], 0
        while True:
            out = np.zeros(max(chunk, 1), self.EVENT_DTYPE)
            n, lost = C.c_uint32(), C.c_uint32()
            self._chk(self._lib.fyx_anim_take_events(self._h, chunk, out.ctypes.data_as(C.c_void_p), C.byref(n), C.byref(lost)))
            parts.append(out[:n.value])
            lost_total += lost.value
            if max_events is not None or n.value < chunk:
                return np.concatenate(parts), lost_total

    def anim_set_root_motion(self, anim: int, node=None, ignore_x=False, ignore_y=False, ignore_z=False, ignore_rotations=False):
        """Animation::set_root_motion_settings: node None = settings None."""
        if node is None:
            self._chk(self._lib.fyx_anim_set_root_motion(self._h, anim, None))
            return
        s = L.fyx_root_motion_settings(int(node), int(bool(ignore_x)), int(bool(ignore_y)), int(bool(ignore_z)), int(bool(ignore_rotations)))
        self._chk(self._lib.fyx_anim_set_root_motion(self._h, anim, C.byref(s)))

    def anim_root_motions(self, first: int, count: int) -> np.ndarray:
        """Animation::root_motion() of `count` animations from `first` (ROOT_MOTION_DTYPE; present = 0 is None)."""
        out = np.zeros(count, self.ROOT_MOTION_DTYPE)
        self._chk(self._lib.fyx_anim_get_root_motions(self._h, first, count, out.ctypes.data_as(C.c_void_p)))
        return out

    def anim_group_root_motions(self, first_group: int, count: int) -> np.ndarray:
        """The final pose's root_motion() of blend groups first_group .. first_group + count (groups count from 1)."""
        out = np.zeros(count, self.ROOT_MOTION_DTYPE)
        self._chk(self._lib.fyx_anim_get_group_root_motions(self._h, first_group, count, out.ctypes.data_as(C.c_void_p)))
        return out

    # ---- N3: draw-prep after the cull ----
    def set_bundle_ids(self, ids, idx=None):
        """Per-node bundle id = dense id of the (material, surface data, render path) key of
        RenderDataBundleStorage::push (renderer/bundle.rs:1253-1257)."""
        ids = np.ascontiguousarray(ids, dtype=np.uint32)
        ix = _u32(idx)
        self._chk(self._lib.fyx_set_bundle_ids(self._h, len(ids), _ptr(ix), _ptr(ids)))

    def set_node_surfaces(self, nodes, surfaces):
        """Mesh::surfaces of the given nodes: surfaces[i] = list of (bundle_id, skin_surface_id or None) for node nodes[i]."""
        idx = np.ascontiguousarray(nodes, dtype=np.uint32)
        first = np.zeros(len(idx) + 1, np.uint32)
        b, sk = [], []
        for i, lst in enumerate(surfaces):
            for bid, sid in lst:
                b.append(bid)
                sk.append(L.FYX_NONE if sid is None else sid)
            first[i + 1] = len(b)
        ba = np.ascontiguousarray(b, dtype=np.uint32)
        sa = np.ascontiguousarray(sk, dtype=np.uint32)
        self._chk(self._lib.fyx_set_node_surfaces(self._h, len(idx), _ptr(idx), _ptr(first), ba.ctypes.data_as(C.c_void_p) if ba.size else None,
                                                  sa.ctypes.data_as(C.c_void_p) if sa.size else None))

    def _instance_surfaces(self, fn, index: int, count: int) -> np.ndarray:
        p = L.u32p()
        self._chk(fn(self._h, index, C.byref(p)))
        return np.ctypeslib.as_array(p, shape=(count,)).copy() if count else np.empty(0, np.uint32)

    def get_instance_surfaces(self, frustum: int, count: int) -> np.ndarray:
        return self._instance_surfaces(self._lib.fyx_get_instance_surfaces, frustum, count)

    def enable_instances(self, enable: bool = True):
        self._chk(self._lib.fyx_enable_instances(self._h, 1 if enable else 0))

    def pack_instances(self, frustum: int, view_m16, view_projection_m16) -> dict:
        """Instances of the frustum's visible list grouped by bundle: dict with node (u32[n]), sort_index (u64[n]),
        world / wvp (f32[n,16], column-major) and bundles (structured array: id, first, count, sort_index)."""
        v = np.ascontiguousarray(view_m16, dtype=np.float32).reshape(16)
        vp = np.ascontiguousarray(view_projection_m16, dtype=np.float32).reshape(16)
        self._chk(self._lib.fyx_pack_instances(self._h, frustum, _ptr(v), _ptr(vp)))
        out = L.fyx_instances()
        self._chk(self._lib.fyx_get_instances(self._h, frustum, C.byref(out)))
        return self._instances_dict(out, self.get_instance_surfaces(frustum, out.count))

    @staticmethod
    def _instances_dict(out: L.fyx_instances, surface: np.ndarray) -> dict:
        n, nb = out.count, out.n_bundles
        bdt = np.dtype([("id", "<u4"), ("first", "<u4"), ("count", "<u4"), ("reserved", "<u4"), ("sort_index", "<u8")])

        def arr(p, dtype, count):
            if count == 0:
                return np.empty(0, dtype=dtype)
            buf = (C.c_char * (count * np.dtype(dtype).itemsize)).from_address(p)
            return np.frombuffer(buf, dtype=dtype, count=count).copy()

        mats = arr(out.matrices, np.float32, n * 32).reshape(n, 2, 16)
        return {
            "surface": surface,
            "node": arr(out.node, np.uint32, n),
            "sort_index": arr(out.sort_index, np.uint64, n),
            "world": mats[:, 0, :].copy(),
            "wvp": mats[:, 1, :].copy(),
            "bundles": arr(out.bundles, bdt, nb),
        }

    # ---- dynamic batching (BatchingMode::Dynamic, scene/mesh/mod.rs:739-753, 804-833) ----
    def add_dynamic_surface(self, node: int, ordinal: int, batch_key: int, layout_id: int, layout, vertices, triangles) -> int:
        """Batch surface `ordinal` of `node` instead of pushing it: layout = (stride, position_offset, normal_offset,
        tangent_offset) with FYX_NONE for an absent attribute, vertices = the VertexBuffer bytes, triangles = (n, 3) u32."""
        ly = L.fyx_dynamic_layout(*[int(x) for x in layout])
        v = np.ascontiguousarray(np.frombuffer(bytes(vertices), np.uint8) if not isinstance(vertices, np.ndarray) else vertices).view(np.uint8)
        t = np.ascontiguousarray(triangles, dtype=np.uint32).reshape(-1, 3)
        if v.size % ly.stride:
            raise ValueError("vertex bytes are not a whole number of records")
        out = C.c_uint32()
        self._chk(self._lib.fyx_add_dynamic_surface(self._h, node, ordinal, batch_key, layout_id, C.byref(ly), v.size // ly.stride,
                                                    v.ctypes.data_as(C.c_void_p) if v.size else None, len(t),
                                                    t.ctypes.data_as(C.c_void_p) if t.size else None, C.byref(out)))
        return out.value

    def clear_dynamic_surfaces(self, nodes=None):
        """Drop the dynamic registrations of `nodes` (None = all)."""
        ix = _u32(nodes)
        self._chk(self._lib.fyx_clear_dynamic_surfaces(self._h, 0 if ix is None else len(ix), _ptr(ix)))

    # fyx_sprite (48 bytes): a Sprite's or dim2::Rectangle's record (scene/sprite.rs:322-405, scene/dim2/rectangle.rs:323-410)
    SPRITE = np.dtype([("kind", "<u4"), ("batch_key", "<u4"), ("layout_id", "<u4"), ("flip", "<u4"), ("uv_rect", "<f4", 4),
                       ("size", "<f4"), ("rotation", "<f4"), ("color", "u1", 4), ("reserved", "<u4")])

    def set_sprites(self, nodes, records):
        """Make `nodes` quad nodes with `records` (SPRITE, one per node), or update their records: kind SPRITE_3D or
        SPRITE_RECTANGLE, flip bit 0 flip_x and bit 1 flip_y.  The packs then batch each as push_triangles does."""
        rec = np.ascontiguousarray(records, dtype=self.SPRITE).reshape(-1)
        ix = _u32(nodes)
        if ix is None or len(ix) != len(rec):
            raise ValueError("one record per node")
        self._chk(self._lib.fyx_set_sprites(self._h, len(rec), _ptr(ix), rec.ctypes.data_as(C.c_void_p)))

    def clear_sprites(self, nodes=None):
        """Make `nodes` (None = every node) ordinary nodes again."""
        ix = _u32(nodes)
        self._chk(self._lib.fyx_clear_sprites(self._h, 0 if ix is None else len(ix), _ptr(ix)))

    DYNAMIC_BUNDLE = np.dtype([("batch_key", "<u4"), ("layout_id", "<u4"), ("first", "<u4"), ("count", "<u4"), ("sort_index", "<u8")])
    DYNAMIC_INSTANCE = np.dtype([("node", "<u4"), ("triangle_offset", "<u4"), ("triangle_count", "<u4"), ("reserved", "<u4")])

    def dynamic_batches(self, kind: str, index: int, device: bool = False) -> dict:
        """The dynamic batches of the last pack of `kind` ("frustum", "shadow" or "observer") for segment `index`: bundles and
        instances (structured arrays) and streams {layout_id: {"stride", "vertices" (u8 bytes), "triangles" ((n, 3) u32)}}.
        device=True reads through the device getter (the same values, copied here)."""
        fn = {"frustum": "fyx_get_dynamic_batches", "shadow": "fyx_get_shadow_dynamic_batches",
              "observer": "fyx_get_scene_observer_dynamic_batches"}[kind] + ("_device" if device else "")
        out = L.fyx_dynamic_batches()
        self._chk(getattr(self._lib, fn)(self._h, index, C.byref(out)))
        if device:
            import torch

            def arr(p, dtype, count):
                if count == 0:
                    return np.empty(0, dtype=dtype)
                nb = count * np.dtype(dtype).itemsize

                class Dev:
                    __cuda_array_interface__ = {"shape": (nb,), "typestr": "|u1", "data": (p, False), "version": 3}

                return torch.as_tensor(Dev(), device="cuda").cpu().numpy().view(dtype)
        else:
            def arr(p, dtype, count):
                if count == 0:
                    return np.empty(0, dtype=dtype)
                buf = (C.c_char * (count * np.dtype(dtype).itemsize)).from_address(p)
                return np.frombuffer(buf, dtype=dtype, count=count).copy()
        streams = {}
        for k in range(out.n_streams):
            st = out.streams[k]
            streams[st.layout_id] = {"stride": st.stride, "vertices": arr(st.vertices, np.uint8, st.n_vertices * st.stride),
                                     "triangles": arr(st.triangles, np.uint32, st.n_triangles * 3).reshape(-1, 3)}
        return {"bundles": arr(out.bundles, self.DYNAMIC_BUNDLE, out.n_bundles),
                "instances": arr(out.instances, self.DYNAMIC_INSTANCE, out.n_instances), "streams": streams}

    def pack_bone_matrices(self, frustum: int):
        """Bone-matrix blocks (255 mat4, zero padded) of the skinned instances of the last pack_instances (bundle.rs:484-496)."""
        self._chk(self._lib.fyx_pack_bone_matrices(self._h, frustum))

    def _bone_matrix_block(self, fn, index: int, instance: int):
        out = np.empty((255, 16), dtype=np.float32)
        has = C.c_uint32()
        self._chk(fn(self._h, index, instance, out.ctypes.data_as(C.c_void_p), C.byref(has)))
        return out if has.value else None

    def get_bone_matrix_block(self, frustum: int, instance: int):
        """(255,16) f32 block of packed instance `instance`, or None for an unskinned instance."""
        return self._bone_matrix_block(self._lib.fyx_get_bone_matrix_block, frustum, instance)

    def pack_shadow_instances(self):
        """Pack the instances of every shadow map of the last cull_shadow_casters (made with enable_instances) in one call;
        read them with get_shadow_instances(map)."""
        self._chk(self._lib.fyx_pack_shadow_instances(self._h))

    def get_shadow_instances(self, map: int) -> dict:
        """Instances of shadow map `map`: the same dict as pack_instances, for the map's observer (its look_at_rh and
        view_projection).  bundles["first"] counts from the map's first instance."""
        out = L.fyx_instances()
        self._chk(self._lib.fyx_get_shadow_instances(self._h, map, C.byref(out)))
        return self._instances_dict(out, self._instance_surfaces(self._lib.fyx_get_shadow_instance_surfaces, map, out.count))

    def pack_shadow_bone_matrices(self):
        """One bone-matrix block (255 mat4, zero padded) per skinned surface, for the last pack_shadow_instances."""
        self._chk(self._lib.fyx_pack_shadow_bone_matrices(self._h))

    def get_shadow_bone_matrix_block(self, map: int, instance: int):
        """(255,16) f32 block of instance `instance` of shadow map `map`, or None for an unskinned instance."""
        return self._bone_matrix_block(self._lib.fyx_get_shadow_bone_matrix_block, map, instance)

    def build_palettes(self):
        self._chk(self._lib.fyx_build_palettes(self._h))

    def skin(self):
        self._chk(self._lib.fyx_skin(self._h))

    def render_prep(self, *, update_flags=L.UPDATE_INCREMENTAL, changed_m16=None, changed_trs=None, changed_rot=None, changed_idx=None, n_changed=None, frusta=(), cam_mask=None,
                    pass_flags=None, do_palettes=True, do_skin=True, readback_visible=True, async_=False, allgather=False,
                    animate_dt=None, readback_own=False):
        """One frame (fyx_render_prep). changed_m16 / changed_idx may be numpy arrays or raw (pinned) addresses."""
        d = L.fyx_frame_desc()
        d.struct_size = C.sizeof(L.fyx_frame_desc)
        d.update_flags = update_flags
        keep = []
        if changed_rot is not None:
            payload, width, field = changed_rot, 4, "changed_rot"
        elif changed_trs is not None:
            payload, width, field = changed_trs, 10, "changed_trs"
        else:
            payload, width, field = changed_m16, 16, "changed_m16"
        if payload is not None:
            if isinstance(payload, np.ndarray):
                m = _f32(payload)
                keep.append(m)
                setattr(d, field, m.ctypes.data)
                d.n_changed = m.size // width if n_changed is None else n_changed
            else:
                setattr(d, field, int(payload))
                d.n_changed = int(n_changed)
            if changed_idx is not None:
                if isinstance(changed_idx, np.ndarray):
                    ix = _u32(changed_idx)
                    keep.append(ix)
                    d.changed_idx = ix.ctypes.data
                else:
                    d.changed_idx = int(changed_idx)
        arr = self._frusta(frusta)
        d.n_frusta = len(frusta)
        d.frusta = C.cast(arr, C.POINTER(L.fyx_frustum))
        cm, pf = _u32(cam_mask), _u32(pass_flags)
        keep += [cm, pf, arr]
        d.cam_mask = None if cm is None else cm.ctypes.data
        d.pass_flags = None if pf is None else pf.ctypes.data
        d.do_palettes = 1 if do_palettes else 0
        d.do_skin = 1 if do_skin else 0
        d.readback_visible = 1 if readback_visible else 0
        d.flags = (L.FRAME_ASYNC if async_ else 0) | (L.FRAME_ALLGATHER if allgather else 0) | (L.FRAME_READBACK_OWN if readback_own else 0)
        if animate_dt is not None:
            d.do_animate = 1
            d.animate_dt = float(animate_dt)
        if async_:
            self._async_keep = keep  # inputs must outlive the enqueued frame
        self._chk(self._lib.fyx_render_prep(self._h, C.byref(d)))

    def frame_wait(self):
        """Collect the oldest pipelined (async + read-back) frame; its visible lists become readable."""
        self._chk(self._lib.fyx_frame_wait(self._h))

    # -- read-back --
    def _gather(self, fn, idx, count, width, dtype):
        idx = _u32(idx)
        n = self.n_nodes if idx is None and count is None else (idx.size if idx is not None else count)
        out = np.empty((n, width) if width > 1 else (n,), dtype=dtype)
        self._chk(fn(self._h, n, _ptr(idx), out.ctypes.data_as(C.c_void_p)))
        return out

    def get_global_matrices(self, idx=None, count=None) -> np.ndarray:
        return self._gather(self._lib.fyx_get_global_matrices, idx, count, 16, np.float32)

    def get_world_aabbs(self, idx=None, count=None) -> np.ndarray:
        return self._gather(self._lib.fyx_get_world_aabbs, idx, count, 6, np.float32)

    def get_global_flags(self, idx=None, count=None) -> np.ndarray:
        return self._gather(self._lib.fyx_get_global_flags, idx, count, 1, np.uint32)

    def get_palette(self, surface_id: int) -> np.ndarray:
        nb = self._surfaces[surface_id][0]
        out = np.empty((nb, 16), dtype=np.float32)
        self._chk(self._lib.fyx_get_palette(self._h, surface_id, out.ctypes.data_as(C.c_void_p)))
        return out

    def get_skinned(self, surface_id: int, normals: bool = True):
        nv = self._surfaces[surface_id][1]
        pos = np.empty((nv, 3), dtype=np.float32)
        nrm = np.empty((nv, 3), dtype=np.float32) if normals else None
        self._chk(self._lib.fyx_get_skinned(self._h, surface_id, pos.ctypes.data_as(C.c_void_p), None if nrm is None else nrm.ctypes.data_as(C.c_void_p)))
        return pos, nrm

    def get_skinned_device(self, surface_id: int):
        p, n = C.c_void_p(), C.c_void_p()
        self._chk(self._lib.fyx_get_skinned_device(self._h, surface_id, C.byref(p), C.byref(n)))
        return p.value, n.value

    def timings(self) -> dict:
        t = L.fyx_timings()
        self._chk(self._lib.fyx_get_timings(self._h, C.byref(t)))
        return {n: getattr(t, n) for n, _ in L.fyx_timings._fields_}

    def kernel_launch_count(self) -> int:
        return int(self._lib.fyx_kernel_launch_count(self._h))

    # -- multi-GPU --
    @staticmethod
    def comm_unique_id() -> bytes:
        buf = C.create_string_buffer(128)
        lib = L.load()
        rc = lib.fyx_comm_get_unique_id(buf)
        if rc != 0:
            raise FyxError(rc, (lib.fyx_last_error(None) or b"").decode())
        return buf.raw

    def comm_init(self, nranks: int, rank: int, uid: bytes):
        assert len(uid) == 128
        self._chk(self._lib.fyx_comm_init(self._h, nranks, rank, C.create_string_buffer(uid, 128)))

    def comm_mode(self) -> str:
        """How the visible lists are exchanged (fyx_comm_mode): decided collectively at the first gathered frame."""
        m = int(self._lib.fyx_comm_mode(self._h))
        if not m:
            return "none"
        if m & L.COMM_UNDECIDED:
            return "nccl initialised, exchange not built yet"
        dev = "peer stores over NVLink (cudaIpc)" if m & L.COMM_PEER_STORES else "ncclAllGather (counts, padded slots, pack kernels)"
        host = "node-wide host segment (each rank copies its own lists)" if m & L.COMM_HOST_SEGMENT else "private copy of the gathered device lists per rank"
        return f"device: {dev}; host: {host}"

    def comm_stats(self) -> dict:
        """The most recent exchange of this rank: entries, NVLink egress bytes, device time (fyx_comm_get_stats)."""
        st = L.fyx_comm_stats()
        self._chk(self._lib.fyx_comm_get_stats(self._h, C.byref(st)))
        return {n: getattr(st, n) for n, _ in L.fyx_comm_stats._fields_}

    def allgather_visible(self):
        self._chk(self._lib.fyx_allgather_visible(self._h))

    def get_visible_gathered(self, frustum: int = 0, copy: bool = True) -> np.ndarray:
        p = L.u32p()
        n = C.c_uint32()
        self._chk(self._lib.fyx_get_visible_gathered(self._h, frustum, C.byref(p), C.byref(n)))
        if n.value == 0:
            return np.empty(0, dtype=np.uint32)
        v = np.ctypeslib.as_array(p, shape=(n.value,))
        return v.copy() if copy else v

    def get_visible_gathered_device(self, frustum: int = 0):
        p = C.c_void_p()
        n = C.c_uint32()
        self._chk(self._lib.fyx_get_visible_gathered_device(self._h, frustum, C.byref(p), C.byref(n)))
        return p.value, n.value
