"""N4 scene observers on the device: fyx_cull_scene_observers against the oracle of ObserversCollection::from_scene and one
from_graph per observer (tests/observer_oracle.py), and against the host route on the device (fyx_set_observers + fyx_cull
on the returned matrices + fyx_cull_lights + fyx_select_reflection_probes, fyx_pack_instances per observer).

The table must equal the oracle's bit for bit (node, kind, face, mask, translation, z range, view, projection,
view_projection); the visible sets, light lists (in pool order) and environment maps must be the oracle's."""
import ctypes as C

import numpy as np
import pytest

import fyrox_b200 as fb
import observer_oracle as oo
import oracle_binding as ob
from fyrox_b200 import _lib as L
from test_gpu_shadow_casters import ShadowScene, local_from_trs, rand_quat
from test_gpu_shadow_csm import same_bits
from test_gpu_shadow_pruned import Pruners

pytestmark = pytest.mark.gpu

f32 = np.float32
FRAME = (1280.0, 720.0)


class ObserverScene:
    """A ShadowScene (lights, masks, rotated and scaled nodes) whose nodes also carry cameras and reflection probes, with LOD
    objects and static batches (Pruners).  Probes get large boxes, so that cameras stand inside some of them."""

    def __init__(self, rng, n, n_cams, n_probes, pruners=True, rotate_all=True):
        self.rng = rng
        self.sc = sc = ShadowScene(rng, n, 12, p_cast=0.5, rotate_all=rotate_all)
        enabled = np.zeros(n, bool)  # globally enabled: parents come before their children
        enabled[0] = True
        on = (sc.flags & fb.NODE_ENABLED) != 0
        for i in range(1, n):
            enabled[i] = enabled[sc.parent[i]] and on[i]
        cand = np.setdiff1d(np.flatnonzero(enabled), np.concatenate([[0], sc.lights]))
        pick = rng.choice(cand, n_cams + n_probes, replace=False)
        self.cam_nodes = np.sort(pick[:n_cams]).astype(np.uint32)
        self.probe_nodes = np.sort(pick[n_cams:]).astype(np.uint32)
        sc.flags[self.probe_nodes] |= np.uint32(fb.NODE_REFLECTION_PROBE)
        sc.aabb[self.probe_nodes] = (-20, -20, -20, 20, 20, 20)
        self.pr = Pruners(sc)
        if pruners:
            self.pr.add_random(rng)
        self.cams, self.probes = {}, {}
        for k, node in enumerate(self.cam_nodes.tolist()):
            ortho = k % 4 == 3
            self.cams[node] = oo.Camera(projection=oo.ORTHOGRAPHIC if ortho else oo.PERSPECTIVE,
                                        fov_or_vertical_size=float(rng.uniform(5, 30) if ortho else rng.uniform(0.5, 1.6)),
                                        z_near=float(rng.uniform(0.05, 1.0)), z_far=float(rng.uniform(30, 150)), enabled=k % 5 != 4,
                                        frame_size=(640.0, 640.0) if k % 3 == 2 else (0.0, 0.0))
        for k, node in enumerate(self.probe_nodes.tolist()):
            self.probes[node] = oo.Probe(update_mode=oo.EACH_FRAME if k % 3 == 0 else oo.ONCE, z_near=float(rng.uniform(0.05, 0.5)),
                                         z_far=float(rng.uniform(10, 60)), rendering_position=tuple(rng.uniform(-1, 1, 3).tolist()))
        self.state = oo.ProbeState()

    def load(self, ctx):
        self.sc.load(ctx)
        self.pr.send_ranges(ctx)
        self.send(ctx)
        return self.pr.oracle()

    def send(self, ctx, cams=None, probes=None):
        cams = self.cams if cams is None else cams
        probes = self.probes if probes is None else probes
        if cams:
            nodes = np.array(sorted(cams), np.uint32)
            rec = np.zeros(len(nodes), fb.Context.CAMERA_DTYPE)
            for k, x in enumerate(nodes.tolist()):
                c = cams[x]
                rec[k] = (int(c.enabled), c.projection, c.fov_or_vertical_size, c.z_near, c.z_far, c.frame_size)
            ctx.set_cameras(nodes, rec)
        if probes:
            nodes = np.array(sorted(probes), np.uint32)
            rec = np.zeros(len(nodes), fb.Context.PROBE_DTYPE)
            for k, x in enumerate(nodes.tolist()):
                p = probes[x]
                rec[k] = (1, p.update_mode, p.z_near, p.z_far, p.rendering_position)
            ctx.set_reflection_probes(nodes, rec)
            self.state.reset(nodes)

    def move(self, ctx, count=40):
        """New TRS records for the observers' parents and some observers themselves, on both sides."""
        sc = self.sc
        obs = np.concatenate([self.cam_nodes, self.probe_nodes])
        idx = np.unique(np.concatenate([sc.parent[obs][sc.parent[obs] != 0xFFFFFFFF], obs[: count // 2]])).astype(np.uint32)
        idx = idx[idx != 0]
        sc.trs[idx, 0:3] += self.rng.uniform(-2, 2, (idx.size, 3)).astype(f32)
        sc.trs[idx, 3:7] = rand_quat(self.rng, idx.size)
        sc.local[idx] = local_from_trs(sc.trs[idx])
        ctx.set_local_trs(sc.trs[idx], idx)
        ctx.update_transforms()
        return self.pr.oracle()


def key(rows):
    return [(int(r["node"]), int(r["kind"]), int(r["face"])) for r in rows]


def observe(ctx, og, s: ObserverScene, frame=FRAME):
    """One call against the oracle; returns (table, entries, lights, oracle observers)."""
    ctx.cull_scene_observers(frame)
    table, entries, lights = ctx.get_scene_observers()
    want = oo.from_scene(og, s.sc.mask, s.cams, s.probes, s.state, frame)
    assert key(table) == [(w["node"], w["kind"], w["face"]) for w in want]
    for r, w in zip(table, want):
        assert int(r["render_mask"]) == w["render_mask"]
        for f in ("translation", "view", "projection", "view_projection"):
            assert same_bits(r[f], w[f]), (f, key([r]))
        assert same_bits(r["z_near"], w["z_near"]) and same_bits(r["z_far"], w["z_far"])
        got = np.sort(entries[r["first"]: r["first"] + r["count"]])
        assert np.array_equal(got, w["visible"]), (key([r]), got.size, w["visible"].size)
        assert np.array_equal(lights[r["lights_first"]: r["lights_first"] + r["lights_count"]], w["lights"])
        assert int(r["environment_map"]) == w["environment_map"]
    return table, entries, lights, want


def host_route(ctx, table):
    """Per 8 observers: fyx_set_observers + fyx_cull on the table's matrices, fyx_cull_lights, fyx_select_reflection_probes."""
    sets, lights, env = [], [], []
    for o0 in range(0, len(table), L.FYX_MAX_FRUSTA):
        rows = table[o0: o0 + L.FYX_MAX_FRUSTA]
        obs = [(r["translation"], float(r["z_near"]), float(r["z_far"])) for r in rows]
        ctx.set_observers(obs)
        fr = [fb.frustum_from_view_projection_matrix(r["view_projection"]) or fb.frustum_default() for r in rows]
        ctx.cull(fr, cam_mask=[int(r["render_mask"]) for r in rows])
        sets += [np.sort(ctx.get_visible(f)) for f in range(len(rows))]
        ctx.cull_lights()
        lights += [ctx.get_visible_lights(f) for f in range(len(rows))]
        env += ctx.select_reflection_probes().tolist()
    return sets, lights, env


def same_as_host_route(ctx, table, entries, lights):
    sets, lts, env = host_route(ctx, table)
    for k, r in enumerate(table):
        assert np.array_equal(np.sort(entries[r["first"]: r["first"] + r["count"]]), sets[k]), key([r])
        assert np.array_equal(lights[r["lights_first"]: r["lights_first"] + r["lights_count"]], lts[k])
        if int(r["kind"]) == oo.CAMERA:
            assert int(r["environment_map"]) == env[k]


@pytest.mark.parametrize("seed", [0, 1])
def test_random_scenes_across_calls(ctx, seed):
    rng = np.random.default_rng(4100 + seed)
    s = ObserverScene(rng, 3000, 6, 4)
    og = s.load(ctx)
    table, entries, lights, want = observe(ctx, og, s)
    assert sum(int(r["kind"]) == oo.PROBE_FACE for r in table) == 24 and len(table) > 24
    assert any(w["environment_map"] != 0xFFFFFFFF for w in want) and any(len(w["lights"]) for w in want)
    lod_vis = [set(w["visible"].tolist()) & set(s.pr.ranges) for w in want]
    assert any(lod_vis) and len({frozenset(v) for v in lod_vis}) > 1  # the LOD filter differs between observers
    same_as_host_route(ctx, table, entries, lights)
    # moved parents: only EachFrame probes come back, then a forced one, then a camera switched off
    og = s.move(ctx)
    observe(ctx, og, s)
    forced = s.probe_nodes[1:2]
    ctx.force_reflection_probe_update(forced)
    s.state.reset(forced)
    t3, _, _, _ = observe(ctx, og, s)
    assert int(forced[0]) in {int(r["node"]) for r in t3}
    c0 = int(s.cam_nodes[0])
    s.cams[c0].enabled = False
    s.send(ctx, cams={c0: s.cams[c0]}, probes={})
    og = s.move(ctx)
    t4, e4, l4, _ = observe(ctx, og, s, frame=(800.0, 1000.0))
    assert c0 not in {int(r["node"]) for r in t4}
    same_as_host_route(ctx, t4, e4, l4)


def test_zero_one_and_many_observers(ctx):
    rng = np.random.default_rng(4200)
    s = ObserverScene(rng, 2500, 3, 12)
    cams, probes = s.cams, s.probes
    s.cams, s.probes = {}, {}
    og = s.load(ctx)
    table, entries, lights, _ = observe(ctx, og, s)
    assert len(table) == 0 and entries.size == 0
    s.cams = {int(s.cam_nodes[0]): cams[int(s.cam_nodes[0])]}
    s.cams[int(s.cam_nodes[0])].enabled = True
    s.send(ctx)
    table, _, _, _ = observe(ctx, og, s)
    assert len(table) == 1
    # every probe EachFrame: 72 faces and the cameras, more than two 32-map pruner words
    s.cams = cams
    s.probes = {k: oo.Probe(oo.EACH_FRAME, p.z_near, p.z_far, p.rendering_position) for k, p in probes.items()}
    s.send(ctx)
    for _ in range(2):
        table, entries, lights, _ = observe(ctx, og, s)
        assert len(table) > 72
    same_as_host_route(ctx, table, entries, lights)


def test_records_carried_across_topology(ctx):
    rng = np.random.default_rng(4300)
    s = ObserverScene(rng, 2000, 4, 3)
    og = s.load(ctx)
    observe(ctx, og, s)
    # the same scene again through fyx_set_topology: records and the probes' rendered bits stay
    s.sc.load(ctx)
    s.pr.send_ranges(ctx)
    t2, _, _, _ = observe(ctx, og, s)
    assert sum(int(r["kind"]) == oo.PROBE_FACE for r in t2) == 6 * sum(p.update_mode == oo.EACH_FRAME for p in s.probes.values())
    # a camera node that a topology removes drops its record: alive again, it is no camera any more
    c = int(s.cam_nodes[0])
    flags = s.sc.flags.copy()
    s.sc.flags[c] &= ~np.uint32(fb.NODE_ALIVE)
    ctx.set_topology(s.sc.parent, s.sc.flags, s.sc.mask, s.sc.aabb)
    s.sc.flags = flags
    s.sc.load(ctx)
    s.pr.send_ranges(ctx)
    ctx.cull_scene_observers(FRAME)
    table, _, _ = ctx.get_scene_observers()
    assert c not in {int(r["node"]) for r in table}
    del s.cams[c]
    observe(ctx, og, s)


def test_instances_against_the_host_route_and_the_oracle(ctx):
    rng = np.random.default_rng(4400)
    s = ObserverScene(rng, 2500, 4, 2)
    ctx.enable_instances(True)
    og = s.load(ctx)
    # palette-only skinned surfaces on some renderable nodes, bones elsewhere in the graph
    sc = s.sc
    renderable = np.flatnonzero((sc.flags & fb.NODE_RENDERABLE) != 0)
    renderable = np.setdiff1d(renderable[renderable > 0], np.concatenate([s.cam_nodes, s.probe_nodes]))
    skinned = set(rng.choice(renderable, 300, replace=False).tolist())
    bone_ib = {}
    for mesh in sorted(skinned):
        bones = rng.choice(np.arange(1, sc.n), int(rng.integers(1, 9)), replace=False).astype(np.uint32)
        for b in bones.tolist():
            if b not in bone_ib:
                ib = np.eye(4, dtype=f32)
                ib[3, 0:3] = rng.uniform(-2, 2, 3)
                bone_ib[b] = ib.reshape(16)
                og.set_inv_bind(b, bone_ib[b])
        og.add_surface(mesh, bones)
        ctx.add_skinned_surface(mesh, bones, np.stack([bone_ib[b] for b in bones.tolist()]), None, n_verts=0)
    og.update_hierarchical_data()
    ctx.update_transforms(fb.UPDATE_ALL)
    ctx.build_palettes()
    table, entries, _, _ = observe(ctx, og, s)
    ctx.pack_scene_observer_instances()
    ctx.pack_scene_observer_bone_matrices()
    n_blocks = 0
    for o, r in enumerate(table):
        got = ctx.get_scene_observer_instances(o)
        assert np.array_equal(np.sort(got["node"]), np.sort(entries[r["first"]: r["first"] + r["count"]]))
        ctx.set_observers([(r["translation"], float(r["z_near"]), float(r["z_far"]))])
        ctx.cull([fb.frustum_from_view_projection_matrix(r["view_projection"]) or fb.frustum_default()], cam_mask=[int(r["render_mask"])])
        want = ctx.pack_instances(0, r["view"], r["view_projection"])
        a, b = np.argsort(got["node"], kind="stable"), np.argsort(want["node"], kind="stable")
        assert np.array_equal(got["node"][a], want["node"][b])
        assert np.array_equal(got["sort_index"][a], want["sort_index"][b])
        assert got["world"][a].tobytes() == want["world"][b].tobytes() and got["wvp"][a].tobytes() == want["wvp"][b].tobytes()
        assert np.array_equal(got["bundles"]["id"], want["bundles"]["id"]) and np.array_equal(got["bundles"]["count"], want["bundles"]["count"])
        plain = [i for i in range(got["node"].size) if int(got["node"][i]) not in skinned]
        for i in plain[:5]:
            si, w, wvp = og.instance(int(got["node"][i]), r["view"], r["view_projection"])
            assert int(got["sort_index"][i]) == si and got["world"][i].tobytes() == w.tobytes() and got["wvp"][i].tobytes() == wvp.tobytes()
        # bone blocks: one per fyx surface, bit for bit write_uniforms' block (renderer/bundle.rs:484-496)
        blocks = BoneBlocks()
        assert ctx._lib.fyx_get_scene_observer_bone_matrix_blocks_device(ctx._h, o, C.byref(blocks)) == 0
        assert blocks.count == got["node"].size and blocks.n_blocks == len(skinned)
        for i in range(got["node"].size):
            nd = int(got["node"][i])
            blk = ctx.get_scene_observer_bone_matrix_block(o, i)
            want_blk = np.empty(255 * 16, f32)
            has = ob.lib().orc_instance_bone_block(og.h, nd, ob.fp(want_blk))
            assert bool(has) == (blk is not None) == (nd in skinned), (o, nd)
            if has:
                assert blk.reshape(-1).tobytes() == want_blk.tobytes(), (o, nd)
                assert got["world"][i].tobytes() == np.eye(4, dtype=f32).reshape(16).tobytes()
                n_blocks += 1
    assert n_blocks > 0
    # a topology makes the slots stale
    s.sc.load(ctx)
    with pytest.raises(fb.FyxError) as e:
        ctx.pack_scene_observer_instances()
    assert e.value.code == L.FYX_ERR_STATE


class BoneBlocks(C.Structure):
    _fields_ = [("count", C.c_uint32), ("n_blocks", C.c_uint32), ("block_of_instance", C.c_void_p), ("blocks", C.c_void_p)]


def test_observers_moved_by_animation(ctx):
    """Cameras, probes and their parents placed by fyx_animate (position tracks) between calls: the observers follow the
    transforms the animation wrote on the device, with no host read-back."""
    rng = np.random.default_rng(4700)
    s = ObserverScene(rng, 2500, 4, 3)
    og = s.load(ctx)
    t0, _, _, _ = observe(ctx, og, s)
    sc = s.sc
    obs = np.concatenate([s.cam_nodes, s.probe_nodes])
    par = sc.parent[obs]
    targets = np.unique(np.concatenate([obs, par[(par != 0xFFFFFFFF) & (par != 0)]])).astype(np.uint32)
    ctx.set_local_trs(sc.trs[targets], targets)  # rotation and scale of these records stay; the animation writes positions
    ctx.update_transforms()
    for step in range(3):
        pos = (sc.trs[targets, 0:3] + rng.uniform(-3, 3, (targets.size, 3))).astype(f32)
        keys = np.zeros(3 * targets.size, fb.Context.KEY_DTYPE)
        tracks = np.zeros(targets.size, fb.Context.TRACK_DTYPE)
        for k, node in enumerate(targets.tolist()):
            for c in range(3):  # one Constant key per curve: the sampled value is the key's, at any time
                keys[3 * k + c] = (0.0, pos[k, c], L.KEY_CONSTANT, 0.0, 0.0)
            tracks[k] = (node, L.BIND_POSITION, L.TV_VECTOR3, 1, 3, (3 * k, 3 * k + 1, 3 * k + 2, 0), (1, 1, 1, 0))
        ctx.anim_clear()
        ctx.anim_add(tracks, keys, time_slice=(0.0, 1.0))
        ctx.animate(0.25)
        ctx.update_transforms()
        sc.trs[targets, 0:3] = pos
        sc.local[targets] = local_from_trs(sc.trs[targets])
        og = s.pr.oracle()
        t1, _, _, _ = observe(ctx, og, s)
        moved = {int(r["node"]): r["translation"].tobytes() for r in t1}
        assert any(moved.get(int(r["node"])) not in (None, r["translation"].tobytes()) for r in t0)
        t0 = t1


def test_one_million_nodes_in_full(ctx):
    rng = np.random.default_rng(4500)
    s = ObserverScene(rng, 1_000_000, 6, 3, rotate_all=False)
    og = s.load(ctx)
    table, entries, lights, _ = observe(ctx, og, s)
    assert len(table) >= 18 and entries.size > 0
    same_as_host_route(ctx, table, entries, lights)


def test_refusals(ctx):
    def code(fn, *a):
        with pytest.raises(fb.FyxError) as e:
            fn(*a)
        return e.value.code

    assert code(ctx.cull_scene_observers, FRAME) == L.FYX_ERR_STATE  # no topology
    rng = np.random.default_rng(4600)
    s = ObserverScene(rng, 500, 2, 1, pruners=False)
    s.load(ctx)
    assert code(ctx.pack_scene_observer_instances) == L.FYX_ERR_STATE  # no observer cull
    for bad in ((0.0, 720.0), (1280.0, -1.0), (np.nan, 1.0)):
        assert code(ctx.cull_scene_observers, bad) == L.FYX_ERR_INVALID_ARGUMENT
    assert ctx._lib.fyx_cull_scene_observers(ctx._h, None) == L.FYX_ERR_INVALID_ARGUMENT
    rec = np.zeros(1, fb.Context.CAMERA_DTYPE)
    rec[0] = (1, 7, 1.0, 0.1, 10.0, (0.0, 0.0))
    assert code(ctx.set_cameras, [1], rec) == L.FYX_ERR_INVALID_ARGUMENT
    rec[0]["projection"] = oo.PERSPECTIVE
    assert code(ctx.set_cameras, [500], rec) == L.FYX_ERR_INVALID_ARGUMENT
    prec = np.zeros(1, fb.Context.PROBE_DTYPE)
    prec[0] = (1, 2, 0.1, 10.0, (0.0, 0.0, 0.0))
    assert code(ctx.set_reflection_probes, [1], prec) == L.FYX_ERR_INVALID_ARGUMENT
    prec[0]["update_mode"] = oo.ONCE
    assert code(ctx.set_reflection_probes, [9999], prec) == L.FYX_ERR_INVALID_ARGUMENT
    assert code(ctx.force_reflection_probe_update, [9999]) == L.FYX_ERR_INVALID_ARGUMENT
    ctx.cull_scene_observers(FRAME)  # made without instances
    assert code(ctx.pack_scene_observer_instances) == L.FYX_ERR_STATE
    assert code(ctx.get_scene_observer_instances, 0) == L.FYX_ERR_STATE
    # a frame in flight
    ctx.render_prep(frusta=[fb.frustum_default()], readback_visible=True, async_=True, do_palettes=False, do_skin=False)
    assert code(ctx.cull_scene_observers, FRAME) == L.FYX_ERR_STATE
    ctx.frame_wait()
    ctx.cull_scene_observers(FRAME)
