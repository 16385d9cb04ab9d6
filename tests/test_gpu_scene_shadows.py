"""N4 shadow maps of the scene's observers on the device: fyx_cull_scene_shadow_casters against the oracle of the shadow loop
run for every observer (tests/observer_shadow_oracle.py), and against the host route on the device (per observer fyx_cull +
fyx_cull_lights + fyx_cull_shadow_casters_pruned with a csm camera built from the observer).

Every observer's refs must be the oracle's maps in order: light, face and cascade identical, view_projection bit for bit,
identical sets.  Rows are numbered in order of first reference; two distinct spot or point rows never share (light, face,
cascade, mask), and a row is only referenced by observers of one mask."""
import ctypes as C

import numpy as np
import pytest

import fyrox_b200 as fb
import observer_oracle as oo
import observer_shadow_oracle as oso
import oracle_binding as ob
from fyrox_b200 import _lib as L
from test_gpu_observers import FRAME, ObserverScene, observe
from test_gpu_shadow_casters import local_from_trs, rand_quat
from test_gpu_shadow_csm import same_bits

pytestmark = pytest.mark.gpu

f32 = np.float32
SETTINGS = (40.0, 40.0, 1, 1)
DIR = fb.LIGHT_DIRECTIONAL


def scene_shadows(ctx, og, s, want, frame=FRAME, settings=SETTINGS, csm=True):
    """One call against the oracle; returns (maps, entries, refs)."""
    ctx.cull_scene_shadow_casters(*settings, csm_enabled=csm)
    maps, entries = ctx.get_shadow_maps()
    refs = ctx.get_scene_shadow_maps()
    per = oso.scene_shadow_maps(og, s.sc.flags, want, s.cams, frame, settings, s.sc.sources, s.sc.scale(), csm_enabled=csm)
    exp = [(o, w) for o, ws in enumerate(per) for w in ws]
    assert len(refs) == len(exp)
    mask_of_row, key_of_row, next_row = {}, {}, 0
    for r, (o, w) in zip(refs, exp):
        assert int(r["observer"]) == o
        k = int(r["map"])
        assert k <= next_row  # rows in order of first reference
        next_row = max(next_row, k + 1)
        m = maps[k]
        assert (int(m["light"]), int(m["face"]), int(m["cascade"])) == (w["light"], w["face"], w["cascade"])
        assert same_bits(m["view_projection"], w["view_projection"]), (o, w["light"], w["face"], w["cascade"])
        got = np.sort(entries[m["first"]: m["first"] + m["count"]])
        assert np.array_equal(got, w["visible"]), (o, w["light"], w["face"], w["cascade"], got.size, w["visible"].size)
        assert mask_of_row.setdefault(k, w["mask"]) == w["mask"]  # the row carries its observers' one mask
        key = (w["light"], w["face"], w["cascade"], w["mask"])
        if s.sc.sources[w["light"]][0] != DIR:
            assert key_of_row.setdefault(key, k) == k  # equal keys: one row
    assert next_row == len(maps)  # every row is referenced
    return maps, entries, refs


WIDE = (200.0, 200.0, 1, 1)


def shadowy(s, radius=25.0, box=40.0):
    """Every light casts shadows and has a large box, so that it sits in many observers' light lists (and in several faces of
    a probe); spot, point and directional records in turn.  Use with the WIDE settings."""
    sc = s.sc
    sc.flags[sc.lights] |= np.uint32(fb.NODE_CAST_SHADOWS)
    sc.aabb[sc.lights] = (-box, -box, -box, box, box, box)
    for k, node in enumerate(sc.lights.tolist()):
        sc.sources[node] = ((fb.LIGHT_SPOT, fb.LIGHT_POINT, fb.LIGHT_POINT, DIR)[k % 4], f32(1.0), f32(radius))


def observe_and_shadow(ctx, og, s, frame=FRAME, csm=True, settings=SETTINGS):
    _, _, _, want = observe(ctx, og, s, frame)
    return want, scene_shadows(ctx, og, s, want, frame, settings=settings, csm=csm)


def move_lights(ctx, s, rng):
    sc = s.sc
    idx = sc.lights[rng.random(sc.lights.size) < 0.5]
    sc.trs[idx, 0:3] += rng.uniform(-3, 3, (idx.size, 3)).astype(f32)
    sc.trs[idx, 3:7] = rand_quat(rng, idx.size)
    sc.local[idx] = local_from_trs(sc.trs[idx])
    ctx.set_local_trs(sc.trs[idx], idx)
    ctx.update_transforms()
    return s.pr.oracle()


@pytest.mark.parametrize("seed", [0, 1])
def test_random_scenes_across_calls(ctx, seed):
    rng = np.random.default_rng(6100 + seed)
    s = ObserverScene(rng, 3000, 6, 4)
    og = s.load(ctx)
    want, (maps, _, refs) = observe_and_shadow(ctx, og, s)
    assert len(maps) < len(refs)  # shared rows
    kinds = {s.sc.sources[int(m["light"])][0] for m in maps}
    assert DIR in kinds and kinds & {fb.LIGHT_SPOT, fb.LIGHT_POINT}
    assert {int(r["observer"]) for r in refs} & {o for o, w in enumerate(want) if w["kind"] == oo.PROBE_FACE}
    scene_shadows(ctx, og, s, want, csm=False)
    scene_shadows(ctx, og, s, want, settings=(15.0, 25.0, 1, 0))
    # lights moved by TRS, the observers' parents moved, then lights placed by fyx_animate
    og = move_lights(ctx, s, rng)
    observe_and_shadow(ctx, og, s)
    og = s.move(ctx)
    observe_and_shadow(ctx, og, s, frame=(800.0, 1000.0))
    sc = s.sc
    targets = sc.lights[:6]
    ctx.set_local_trs(sc.trs[targets], targets)
    pos = (sc.trs[targets, 0:3] + rng.uniform(-3, 3, (targets.size, 3))).astype(f32)
    keys = np.zeros(3 * targets.size, fb.Context.KEY_DTYPE)
    tracks = np.zeros(targets.size, fb.Context.TRACK_DTYPE)
    for k, node in enumerate(targets.tolist()):
        for c in range(3):
            keys[3 * k + c] = (0.0, pos[k, c], L.KEY_CONSTANT, 0.0, 0.0)
        tracks[k] = (node, L.BIND_POSITION, L.TV_VECTOR3, 1, 3, (3 * k, 3 * k + 1, 3 * k + 2, 0), (1, 1, 1, 0))
    ctx.anim_add(tracks, keys, time_slice=(0.0, 1.0))
    ctx.animate(0.25)
    ctx.update_transforms()
    sc.trs[targets, 0:3] = pos
    sc.local[targets] = local_from_trs(sc.trs[targets])
    observe_and_shadow(ctx, s.pr.oracle(), s)


def test_distinct_masks_are_not_merged(ctx):
    rng = np.random.default_rng(6200)
    s = ObserverScene(rng, 2500, 4, 2)
    obs = np.concatenate([s.cam_nodes, s.probe_nodes])
    s.sc.mask[obs] = (1 << np.arange(obs.size)).astype(np.uint32)
    s.probes = {k: oo.Probe(oo.EACH_FRAME, p.z_near, p.z_far, p.rendering_position) for k, p in s.probes.items()}
    shadowy(s)
    og = s.load(ctx)
    want, (maps, _, refs) = observe_and_shadow(ctx, og, s, settings=WIDE)
    masks = {int(w["render_mask"]) for w in want}
    assert len(masks) > 2
    by_row = {}
    for r in refs:
        by_row.setdefault(int(r["map"]), set()).add(int(want[int(r["observer"])]["render_mask"]))
    assert all(len(v) == 1 for v in by_row.values())
    assert len(maps) < len(refs)  # the faces of one probe still share


def test_zero_observers_no_lights_and_many_candidates(ctx):
    rng = np.random.default_rng(6300)
    s = ObserverScene(rng, 2500, 3, 12)
    shadowy(s)
    cams, probes = s.cams, s.probes
    s.cams, s.probes = {}, {}
    og = s.load(ctx)
    _, (maps, entries, refs) = observe_and_shadow(ctx, og, s, settings=WIDE)
    assert len(maps) == 0 and len(refs) == 0 and entries.size == 0
    # every probe EachFrame: 72 faces and the cameras; candidates cross a 256-wide scan block, maps fill several pruner words
    s.cams = cams
    s.probes = {k: oo.Probe(oo.EACH_FRAME, p.z_near, 200.0, p.rendering_position) for k, p in probes.items()}
    s.send(ctx)
    for _ in range(2):
        want, (maps, _, refs) = observe_and_shadow(ctx, og, s, settings=WIDE)
        assert len(want) > 72 and sum(len(w["lights"]) for w in want) > 256 and len(maps) > 64
    # observers whose light lists are empty: no light node
    flags = s.sc.flags.copy()
    s.sc.flags[s.sc.lights] &= ~np.uint32(fb.NODE_LIGHT)
    og = s.load(ctx)
    want, (maps, _, refs) = observe_and_shadow(ctx, og, s, settings=WIDE)
    assert len(want) > 0 and all(len(w["lights"]) == 0 for w in want) and len(refs) == 0
    s.sc.flags = flags


class BoneBlocks(C.Structure):
    _fields_ = [("count", C.c_uint32), ("n_blocks", C.c_uint32), ("block_of_instance", C.c_void_p), ("blocks", C.c_void_p)]


def test_instances_and_bone_blocks(ctx):
    rng = np.random.default_rng(6400)
    s = ObserverScene(rng, 2500, 4, 2)
    ctx.enable_instances(True)
    og = s.load(ctx)
    sc = s.sc
    renderable = np.flatnonzero((sc.flags & fb.NODE_RENDERABLE) != 0)
    renderable = renderable[renderable > 0]
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
    _, (maps, entries, refs) = observe_and_shadow(ctx, og, s)
    ctx.pack_shadow_instances()
    ctx.pack_shadow_bone_matrices()
    n_blocks = 0
    views = {}
    for r in refs:
        views.setdefault(int(r["map"]), None)
    for k in sorted(views):
        m = maps[k]
        got = ctx.get_shadow_instances(k)
        assert np.array_equal(np.sort(got["node"]), np.sort(entries[m["first"]: m["first"] + m["count"]]))
        blocks = BoneBlocks()
        assert ctx._lib.fyx_get_shadow_bone_matrix_blocks_device(ctx._h, k, C.byref(blocks)) == 0
        assert blocks.count == got["node"].size
        for i in range(min(got["node"].size, 40)):
            nd = int(got["node"][i])
            blk = ctx.get_shadow_bone_matrix_block(k, i)
            want_blk = np.empty(255 * 16, f32)
            has = ob.lib().orc_instance_bone_block(og.h, nd, ob.fp(want_blk))
            assert bool(has) == (blk is not None) == (nd in skinned), (k, nd)
            if has:
                assert blk.reshape(-1).tobytes() == want_blk.tobytes(), (k, nd)
                n_blocks += 1
            else:
                # a plain instance: world and wvp as og.instance gives them for the map's view_projection
                _, w, wvp = og.instance(nd, np.eye(4, dtype=f32).reshape(16), m["view_projection"])
                assert got["world"][i].tobytes() == w.tobytes() and got["wvp"][i].tobytes() == wvp.tobytes()
    assert n_blocks > 0


def host_route(ctx, table, s, frame=FRAME, settings=SETTINGS):
    """Per observer: fyx_cull on its frustum and mask, fyx_cull_lights, fyx_cull_shadow_casters_pruned with a csm camera
    built from it.  Returns per observer [(light, face, cascade, view_projection bytes, sorted set)]."""
    out = []
    ctx.set_observers([])
    for r in table:
        ctx.cull([fb.frustum_from_view_projection_matrix(r["view_projection"]) or fb.frustum_default()], cam_mask=[int(r["render_mask"])])
        ctx.cull_lights()
        if int(r["kind"]) == oo.CAMERA:
            c = s.cams[int(r["node"])]
            fs = c.frame_size if c.frame_size != (0.0, 0.0) else frame
            kw = dict(fov=c.fov_or_vertical_size) if c.projection == oo.PERSPECTIVE else dict(vertical_size=c.fov_or_vertical_size)
            cam = fb.Context.csm_camera(r["view"], fs, float(r["z_near"]), float(r["z_far"]), **kw)
        else:
            cam = fb.Context.csm_camera(r["view"], (1.0, 1.0), float(r["z_near"]), float(r["z_far"]), fov=float(oo.FOV_90))
        ctx.cull_shadow_casters(0, r["translation"], *settings, csm_camera=cam, prune=True)
        maps, entries = ctx.get_shadow_maps()
        out.append([(int(m["light"]), int(m["face"]), int(m["cascade"]), m["view_projection"].tobytes(),
                     np.sort(entries[m["first"]: m["first"] + m["count"]])) for m in maps])
    return out


def test_one_million_nodes_against_the_host_route(ctx):
    rng = np.random.default_rng(6500)
    s = ObserverScene(rng, 1_000_000, 2, 1, rotate_all=False)
    shadowy(s)
    s.load(ctx)
    ctx.cull_scene_observers(FRAME)
    table, _, _ = ctx.get_scene_observers()
    ctx.cull_scene_shadow_casters(*WIDE)
    maps, entries = ctx.get_shadow_maps()
    refs = ctx.get_scene_shadow_maps()
    dev = [[] for _ in range(len(table))]
    for r in refs:
        m = maps[int(r["map"])]
        dev[int(r["observer"])].append((int(m["light"]), int(m["face"]), int(m["cascade"]), m["view_projection"].tobytes(),
                                        np.sort(entries[m["first"]: m["first"] + m["count"]])))
    host = host_route(ctx, table, s, settings=WIDE)
    assert len(refs) > len(maps) and sum(len(x[4]) for d in dev for x in d) > 0
    for d, h in zip(dev, host):
        assert [x[:4] for x in d] == [x[:4] for x in h]
        assert all(np.array_equal(a[4], b[4]) for a, b in zip(d, h))


def test_refusals(ctx):
    def code(fn, *a, **kw):
        with pytest.raises(fb.FyxError) as e:
            fn(*a, **kw)
        return e.value.code

    st = L.fyx_shadow_settings(10.0, 10.0, 1, 1)
    assert ctx._lib.fyx_cull_scene_shadow_casters(None, C.byref(st), 1) == L.FYX_ERR_INVALID_ARGUMENT
    assert ctx._lib.fyx_cull_scene_shadow_casters(ctx._h, None, 1) == L.FYX_ERR_INVALID_ARGUMENT
    assert code(ctx.cull_scene_shadow_casters) == L.FYX_ERR_STATE  # no topology
    rng = np.random.default_rng(6600)
    s = ObserverScene(rng, 800, 2, 1, pruners=False)
    og = s.load(ctx)
    assert code(ctx.cull_scene_shadow_casters) == L.FYX_ERR_STATE  # no observer cull
    assert code(ctx.get_scene_shadow_maps) == L.FYX_ERR_STATE
    want, _ = observe_and_shadow(ctx, og, s)
    # a later single-camera shadow cull replaces the result
    ctx.cull([fb.frustum_default()])
    ctx.cull_shadow_casters(0, np.zeros(3, f32))
    assert code(ctx.get_scene_shadow_maps) == L.FYX_ERR_STATE
    assert code(ctx.get_scene_shadow_maps_device) == L.FYX_ERR_STATE
    # a hierarchy update or a topology since the observer call
    ctx.update_transforms()
    assert code(ctx.cull_scene_shadow_casters) == L.FYX_ERR_STATE
    ctx.cull_scene_observers(FRAME)
    ctx.cull_scene_shadow_casters()
    s.sc.load(ctx)
    assert code(ctx.cull_scene_shadow_casters) == L.FYX_ERR_STATE
    ctx.cull_scene_observers(FRAME)
    ctx.cull_scene_shadow_casters()
    # a frame in flight
    ctx.render_prep(frusta=[fb.frustum_default()], readback_visible=True, async_=True, do_palettes=False, do_skin=False)
    assert code(ctx.cull_scene_shadow_casters) == L.FYX_ERR_STATE
    ctx.frame_wait()
    assert code(ctx.cull_scene_shadow_casters) == L.FYX_ERR_STATE  # the frame updated the hierarchy
    ctx.cull_scene_observers(FRAME)
    ctx.cull_scene_shadow_casters()
    p, n = ctx.get_scene_shadow_maps_device()
    assert p and n == len(ctx.get_scene_shadow_maps())
    assert ctx._lib.fyx_get_scene_shadow_maps(ctx._h, None, None) == L.FYX_ERR_INVALID_ARGUMENT
    assert ctx._lib.fyx_get_scene_shadow_maps_device(None, None, None) == L.FYX_ERR_INVALID_ARGUMENT
