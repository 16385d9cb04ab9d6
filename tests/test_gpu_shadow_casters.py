"""N4 shadow casters on the device: fyx_cull_shadow_casters against the oracle of the deferred light renderer's shadow-map loop
(tests/shadow_oracle.py: renderer/light.rs:509-606, 695-763; shadow/spot.rs:142, shadow/point.rs:162-180).

Map tables (light, face, cascade) must equal the oracle's, view_projection bit for bit, and every map's list must be the set
the oracle's from_graph(map frustum, camera mask, shadow pass) returns."""
import ctypes as C

import numpy as np
import pytest

import fyrox_b200 as fb
import oracle_binding as ob
import shadow_oracle as so
from fyrox_b200 import _lib as L
from helpers import NONE, camera_frustum

pytestmark = pytest.mark.gpu

f32 = np.float32
RENDER = fb.NODE_DEFAULT | fb.NODE_RENDERABLE
SETTINGS = (40.0, 40.0, 1, 1)


def rand_quat(rng, n):
    q = rng.normal(size=(n, 4)).astype(f32)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    return q


def local_from_trs(trs):
    """orc_transform_calculate_local (scene/transform.rs:421-540) of TRS rows with default statics."""
    out = np.empty((len(trs), 16), f32)
    t = ob.Transform()
    for i in range(len(trs)):
        ob.lib().orc_transform_identity(C.byref(t))
        t.local_position[:] = trs[i, 0:3].tolist()
        t.local_rotation[:] = trs[i, 3:7].tolist()
        t.local_scale[:] = trs[i, 7:10].tolist()
        ob.lib().orc_transform_calculate_local(C.byref(t), ob.fp(out[i]))
    return out


class ShadowScene:
    """Root 0; every other node hangs from the root or (30 %) from an earlier node.  Lights carry TRS records (rotated,
    scaled); the other nodes translation-only local matrices (rotated too where `rotate_all`).  Both sides load the same."""

    def __init__(self, rng, n, n_lights, spread=30.0, depth_z=(-70.0, 10.0), rotate_all=True, kinds=(1, 2, 3), p_cast=0.8):
        self.n = n
        parent = np.zeros(n, np.uint32)
        parent[0] = NONE
        nested = rng.random(n) < 0.3
        earlier = (rng.random(n) * np.arange(n)).astype(np.uint32)
        parent[1:] = np.where(nested[1:], earlier[1:], 0)
        flags = np.full(n, RENDER, np.uint32)
        flags[0] = fb.NODE_DEFAULT
        r = rng.random((n, 4))
        flags[1:] &= ~np.where(r[1:, 0] < 0.03, fb.NODE_VISIBILITY, 0).astype(np.uint32)
        flags[1:] &= ~np.where(r[1:, 1] < 0.03, fb.NODE_ENABLED, 0).astype(np.uint32)
        flags[1:] &= ~np.where(r[1:, 2] < 1.0 - p_cast, fb.NODE_CAST_SHADOWS, 0).astype(np.uint32)
        flags[1:] &= ~np.where(r[1:, 3] < 0.05, fb.NODE_FRUSTUM_CULLING, 0).astype(np.uint32)
        self.mask = np.where(rng.random(n) < 0.85, 0xFFFFFFFF, 1 << rng.integers(0, 3, n)).astype(np.uint32)
        pos = np.empty((n, 3), f32)
        pos[:, 0:2] = rng.uniform(-spread, spread, (n, 2))
        pos[:, 2] = rng.uniform(depth_z[0], depth_z[1], n)
        pos[nested] *= f32(0.15)  # children stay near their parent
        self.trs = np.zeros((n, 10), f32)
        self.trs[:, 0:3] = pos
        self.trs[:, 3:7] = rand_quat(rng, n) if rotate_all else (0, 0, 0, 1)
        self.trs[:, 7:10] = 1.0
        self.lights = np.sort(rng.choice(np.arange(1, n), n_lights, replace=False)).astype(np.uint32)
        self.trs[self.lights, 3:7] = rand_quat(rng, n_lights)
        self.trs[self.lights, 7:10] = rng.uniform(0.5, 2.0, (n_lights, 3))
        self.trs[0] = (0, 0, 0, 0, 0, 0, 1, 1, 1, 1)
        flags[self.lights] |= fb.NODE_LIGHT
        self.flags = flags
        self.parent = parent
        if rotate_all:
            self.local = local_from_trs(self.trs)
        else:
            self.local = np.tile(np.eye(4, dtype=f32).reshape(16), (n, 1))
            self.local[:, 12:15] = pos
            self.local[0, 12:15] = 0
            self.local[self.lights] = local_from_trs(self.trs[self.lights])
        h = rng.uniform(0.2, 2.0, (n, 3)).astype(f32)
        self.aabb = np.concatenate([-h, h], axis=1)
        self.sources = {}
        for node in self.lights.tolist():
            kind = int(rng.choice(kinds))
            self.sources[node] = (kind, f32(rng.uniform(0.3, 2.2)), f32(rng.uniform(2.0, 25.0)))

    def load(self, ctx):
        og = ob.Graph.build(self.parent, self.flags, self.mask, self.local, self.aabb)
        og.update_hierarchical_data()
        ctx.set_topology(self.parent, self.flags, self.mask, self.aabb)
        ctx.set_local_matrices(self.local)
        ctx.set_local_trs(self.trs[self.lights], self.lights)  # the lights' scale comes from their TRS records
        ctx.update_transforms(fb.UPDATE_ALL)
        self.send_sources(ctx, self.sources)
        return og

    @staticmethod
    def send_sources(ctx, sources):
        nodes = np.array(sorted(sources), np.uint32)
        rec = np.zeros(len(nodes), fb.Context.LIGHT_SOURCE_DTYPE)
        for k, node in enumerate(nodes.tolist()):
            rec[k] = sources[node]
        ctx.set_light_sources(rec, nodes)

    def scale(self):
        return {int(i): tuple(self.trs[i, 7:10].tolist()) for i in self.lights}


def compare(ctx, og, sc, eye=(0.0, 0.0, 0.0), target=(0.0, 0.0, -1.0), cam_mask=0xFFFFFFFF, settings=SETTINGS, frustum=0, extra=()):
    """Cull the camera (plus `extra` frusta), run the shadow cull and compare everything with the oracle."""
    fo, ff = camera_frustum(eye, target, zfar=150.0)
    frusta = list(extra) + [ff] if frustum else [ff] + list(extra)
    ctx.cull(frusta, cam_mask=[cam_mask] * len(frusta))
    ctx.cull_shadow_casters(frustum, np.array(eye, f32), *settings)
    maps, entries = ctx.get_shadow_maps()
    want = so.shadow_maps(og, sc.flags, fo, eye, cam_mask, settings, sc.sources, sc.scale())
    assert [(int(m["light"]), int(m["face"]), int(m["cascade"])) for m in maps] == [(w[0], w[1], w[2]) for w in want]
    for m, w in zip(maps, want):
        assert m["view_projection"].tobytes() == w[3].tobytes(), (int(m["light"]), int(m["face"]))
        got = np.sort(entries[m["first"]: m["first"] + m["count"]])
        assert np.array_equal(got, w[4]), (int(m["light"]), int(m["face"]), len(got), len(w[4]))
    return maps, entries


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_random_scenes_match_the_oracle(ctx, seed):
    rng = np.random.default_rng(700 + seed)
    sc = ShadowScene(rng, 4000, 40)
    og = sc.load(ctx)
    maps, _ = compare(ctx, og, sc)
    assert len(maps) > 0
    # another camera: moved, turned, a render mask that drops some nodes, different settings; camera frustum not first
    _, f2 = camera_frustum((0, 0, 0), (1, 0, 0))
    compare(ctx, og, sc, eye=(3.0, 1.0, -10.0), target=(2.0, 0.5, -11.0), cam_mask=0x1, settings=(25.0, 60.0, 1, 1), frustum=1, extra=[f2])
    compare(ctx, og, sc, settings=(40.0, 40.0, 0, 1))
    compare(ctx, og, sc, settings=(40.0, 40.0, 1, 0))


def test_lights_moved_between_frames_by_trs_and_animate(ctx):
    rng = np.random.default_rng(71)
    sc = ShadowScene(rng, 2000, 12, kinds=(1, 2))
    og = sc.load(ctx)
    compare(ctx, og, sc)
    # frame 2: fyx_set_local_trs moves, turns and rescales half of the lights
    moved = sc.lights[::2]
    sc.trs[moved, 0:3] += rng.uniform(-6, 6, (len(moved), 3)).astype(f32)
    sc.trs[moved, 3:7] = rand_quat(rng, len(moved))
    sc.trs[moved, 7:10] = rng.uniform(0.5, 2.5, (len(moved), 3)).astype(f32)
    loc = local_from_trs(sc.trs[moved])
    for i, node in enumerate(moved.tolist()):
        og.set_local_matrix(node, loc[i])
    og.update()
    ctx.set_local_trs(sc.trs[moved], moved)
    ctx.update_transforms(fb.UPDATE_INCREMENTAL)
    compare(ctx, og, sc)
    # frames 3..: fyx_animate drives position and scale of other lights; nothing is read back between the frames
    animated = sc.lights[1::2][:4]
    keys, tracks = [], []
    for node in animated.tolist():
        for binding, base in ((ob.BIND_POSITION, sc.trs[node, 0:3]), (ob.BIND_SCALE, sc.trs[node, 7:10])):
            t = np.zeros((), ob.TRACK_DTYPE)
            t["target_node"], t["binding"], t["value_kind"], t["enabled"], t["n_curves"] = node, binding, ob.TV_VECTOR3, 1, 3
            for c in range(3):
                t["first_key"][c], t["n_keys"][c] = len(keys), 2
                v0 = float(base[c])
                keys.append((0.0, v0, 1, 0.0, 0.0))
                keys.append((2.0, v0 + float(rng.uniform(-4, 4)) if binding == ob.BIND_POSITION else float(rng.uniform(0.5, 2.5)), 1, 0.0, 0.0))
            tracks.append(t)
    tk = np.array(tracks, ob.TRACK_DTYPE)
    kk = np.zeros(len(keys), ob.KEY_DTYPE)
    for i, k in enumerate(keys):
        kk[i] = k
    anim = ob.Animation(tk, kk, looped=True, time_slice=(0.0, 2.0))
    ctx.anim_add(tk, kk, looped=True, time_slice=(0.0, 2.0))
    arr = (ob.Transform * sc.n)()
    for i in range(sc.n):
        ob.lib().orc_transform_identity(C.byref(arr[i]))
    for node in sc.lights.tolist():
        t = arr[node]
        t.local_position[:] = sc.trs[node, 0:3].tolist()
        t.local_rotation[:] = sc.trs[node, 3:7].tolist()
        t.local_scale[:] = sc.trs[node, 7:10].tolist()
    for frame in range(3):
        ob.update_animations([anim], 0.375, og, arr)
        og.update()
        ctx.animate(0.375)
        ctx.update_transforms(fb.UPDATE_INCREMENTAL)
        for node in animated.tolist():
            sc.trs[node, 0:3] = list(arr[node].local_position)
            sc.trs[node, 7:10] = list(arr[node].local_scale)
        compare(ctx, og, sc)


def in_view(rng, sc):
    """Hang every light from the root, visible, enabled and casting, well inside the camera's view."""
    for node in sc.lights.tolist():
        sc.flags[node] = RENDER | fb.NODE_LIGHT
        z = rng.uniform(-30.0, -6.0)
        sc.trs[node, 0:3] = (rng.uniform(-0.3, 0.3) * -z, rng.uniform(-0.3, 0.3) * -z, z)
    sc.parent[sc.lights] = 0
    sc.local[sc.lights] = local_from_trs(sc.trs[sc.lights])


def test_zero_one_many_and_very_many_maps(ctx):
    rng = np.random.default_rng(72)
    sc = ShadowScene(rng, 3000, 60, spread=12.0, depth_z=(-30.0, -2.0), kinds=(2,), p_cast=1.0)
    in_view(rng, sc)
    og = sc.load(ctx)
    all_sources = dict(sc.sources)
    big = (200.0, 200.0, 1, 1)
    maps, _ = compare(ctx, og, sc, settings=big)
    assert len(maps) > 256
    # more than 32 maps
    sc.sources = {k: all_sources[k] for k in sorted(all_sources)[:7]}
    ShadowScene.send_sources(ctx, {k: (fb.LIGHT_UNKNOWN, 0.0, 0.0) for k in sorted(all_sources)[7:]})
    maps, _ = compare(ctx, og, sc, settings=big)
    assert 32 < len(maps) <= 42
    # one map: a single spot light
    first = sorted(all_sources)[0]
    sc.sources = {first: (fb.LIGHT_SPOT, f32(1.0), f32(10.0))}
    ShadowScene.send_sources(ctx, {k: (fb.LIGHT_UNKNOWN, 0.0, 0.0) for k in sorted(all_sources)})
    ShadowScene.send_sources(ctx, sc.sources)
    maps, _ = compare(ctx, og, sc, settings=big)
    assert len(maps) == 1
    # zero maps: shadows off for both kinds, then no records at all
    maps, entries = compare(ctx, og, sc, settings=(200.0, 200.0, 0, 0))
    assert len(maps) == 0 and len(entries) == 0
    sc.sources = {}
    ShadowScene.send_sources(ctx, {first: (fb.LIGHT_UNKNOWN, 0.0, 0.0)})
    maps, _ = compare(ctx, og, sc, settings=big)
    assert len(maps) == 0


def test_one_million_nodes_forty_maps_compared_in_full(ctx):
    rng = np.random.default_rng(73)
    sc = ShadowScene(rng, 1_000_000, 20, spread=40.0, rotate_all=False, kinds=(1, 2), p_cast=1.0)
    in_view(rng, sc)
    for node in sc.lights.tolist():
        sc.sources[node] = (fb.LIGHT_POINT if node % 3 else fb.LIGHT_SPOT, f32(1.2), f32(rng.uniform(4.0, 12.0)))
    og = sc.load(ctx)
    maps, entries = compare(ctx, og, sc, settings=(200.0, 200.0, 1, 1))
    assert len(maps) >= 40 and len(entries) > 10_000


def test_fyx_cull_with_the_returned_matrices_gives_the_same_sets(ctx):
    rng = np.random.default_rng(74)
    sc = ShadowScene(rng, 5000, 30)
    og = sc.load(ctx)
    maps, entries = compare(ctx, og, sc)
    assert len(maps) > 8
    lists = [np.sort(entries[m["first"]: m["first"] + m["count"]]) for m in maps]
    vps = [m["view_projection"].copy() for m in maps]
    for b in range(0, len(vps), 8):
        chunk = vps[b: b + 8]
        frusta = [fb.frustum_from_view_projection_matrix(vp) or fb.frustum_default() for vp in chunk]
        ctx.cull(frusta, cam_mask=[0xFFFFFFFF] * len(frusta), pass_flags=[fb.PASS_SHADOW] * len(frusta))
        for k in range(len(chunk)):
            assert np.array_equal(np.sort(ctx.get_visible(k)), lists[b + k])


def code_of(fn):
    with pytest.raises(fb.FyxError) as e:
        fn()
    return e.value.code


def test_state_and_argument_errors(ctx):
    rng = np.random.default_rng(75)
    sc = ShadowScene(rng, 500, 6)
    og = sc.load(ctx)
    t = np.zeros(3, f32)
    assert code_of(lambda: ctx.cull_shadow_casters(0, t)) == L.FYX_ERR_STATE  # no cull yet
    assert code_of(lambda: ctx.get_shadow_maps()) == L.FYX_ERR_STATE
    _, ff = camera_frustum(zfar=150.0)
    ctx.cull([ff, ff])
    assert code_of(lambda: ctx.cull_shadow_casters(2, t)) == L.FYX_ERR_INVALID_ARGUMENT
    ctx.cull_shadow_casters(1, t)
    # a frame in flight
    ctx.render_prep(frusta=[ff], async_=True, readback_visible=True, do_palettes=False, do_skin=False)
    assert code_of(lambda: ctx.cull_shadow_casters(0, t)) == L.FYX_ERR_STATE
    ctx.frame_wait()
    ctx.cull_shadow_casters(0, t)
    # LOD ranges with observers
    ctx.set_lod_ranges(np.array([0.0, 0.5], f32), np.array([int(sc.lights[0])], np.uint32))
    ctx.set_observers([((0, 0, 0), 0.1, 150.0)])
    ctx.cull([ff])
    assert code_of(lambda: ctx.cull_shadow_casters(0, t)) == L.FYX_ERR_STATE
    ctx.set_observers([])
    ctx.cull([ff])
    ctx.cull_shadow_casters(0, t)
    # a statically batched mesh
    flags = sc.flags.copy()
    flags[5] |= fb.NODE_STATIC_BATCH
    ctx.set_flags(flags[5:6], np.array([5], np.uint32))
    ctx.update_transforms(fb.UPDATE_ALL)
    ctx.cull([ff])
    assert code_of(lambda: ctx.cull_shadow_casters(0, t)) == L.FYX_ERR_STATE
    # argument checks of the record call
    bad = np.zeros(1, fb.Context.LIGHT_SOURCE_DTYPE)
    bad["kind"] = 9
    assert code_of(lambda: ctx.set_light_sources(bad, np.array([1], np.uint32))) == L.FYX_ERR_INVALID_ARGUMENT
    ok = np.zeros(1, fb.Context.LIGHT_SOURCE_DTYPE)
    assert code_of(lambda: ctx.set_light_sources(ok, np.array([sc.n], np.uint32))) == L.FYX_ERR_INVALID_ARGUMENT
    del og
