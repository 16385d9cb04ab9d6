"""Cascaded shadow maps of directional lights on the device: fyx_cull_shadow_casters_csm against tests/csm_oracle.py
(renderer/shadow/csm.rs:165-277, gating renderer/light.rs:555-565), in one table with the spot and point maps.

Map tables (light, face, cascade) must equal the oracle's, view_projection bit for bit, and every map's list must be the set
the oracle's from_graph(map frustum, camera mask, shadow pass) returns."""
import ctypes as C

import numpy as np
import pytest

import csm_oracle as co
import fyrox_b200 as fb
import oracle_binding as ob
import shadow_oracle as so
from fyrox_b200 import _lib as L
from helpers import camera_frustum
from test_gpu_shadow_casters import ShadowScene, in_view, local_from_trs, rand_quat
from test_gpu_shadow_instances import check_map, map_view, with_bundles

pytestmark = pytest.mark.gpu

f32 = np.float32
SETTINGS = (40.0, 40.0, 1, 1)
DIR = fb.LIGHT_DIRECTIONAL


def camera(kind=co.PERSPECTIVE, eye=(0.0, 0.0, 0.0), target=(0.0, 0.0, -1.0), z_near=0.1, z_far=150.0, frame=(1920.0, 1080.0), size=None,
           enabled=True):
    """(oracle camera frustum, fyx frustum, oracle CsmCamera, fyx_csm_camera) of one camera; the cull frustum is the camera's
    own projection · view."""
    view = ob.look_at_rh(eye, target, (0.0, 1.0, 0.0))
    fov = float(np.deg2rad(60.0))
    oc = co.CsmCamera(kind, fov if kind == co.PERSPECTIVE else size, z_near, z_far, frame, view, enabled)
    vp = ob.mat4_mul(co.projection_matrix(oc, z_near, z_far), view)
    fo = ob.frustum_from_vp(vp)
    ff = fb.frustum_from_view_projection_matrix(vp)
    if fo is None or ff is None:  # a projection without a frustum: the light list comes from a regular camera
        fo, ff = camera_frustum(eye, target, zfar=150.0)
    if kind == co.PERSPECTIVE:
        fc = fb.Context.csm_camera(view, frame, z_near, z_far, fov=fov, csm_enabled=enabled)
    else:
        fc = fb.Context.csm_camera(view, frame, z_near, z_far, vertical_size=size, csm_enabled=enabled)
    return fo, ff, oc, fc


def send_options(ctx, oc, options):
    """The same split options to the context and the oracle camera."""
    oc.options = dict(options)
    if not options:
        return
    nodes = np.array(sorted(options), np.uint32)
    rec = np.zeros(len(nodes), fb.Context.CSM_OPTIONS_DTYPE)
    for k, node in enumerate(nodes.tolist()):
        rec[k] = (options[node][0], options[node][1])
    ctx.set_csm_options(rec, nodes)


def random_options(rng, lights, relative):
    out = {}
    for node in lights:
        if relative:
            out[int(node)] = (1, tuple(np.sort(rng.uniform(0.02, 1.0, 3)).tolist()))
        else:
            out[int(node)] = (0, tuple(np.sort(rng.uniform(1.0, 120.0, 3)).tolist()))
    return out


def same_bits(a, b):
    """Bit for bit, except that any NaN equals any NaN (the payload of a NaN the arithmetic makes is the platform's choice:
    a frame with h = 0 gives the reference NaN matrices too)."""
    a, b = np.asarray(a, f32), np.asarray(b, f32)
    return bool(np.all((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))))


def compare(ctx, og, sc, cam, eye=(0.0, 0.0, 0.0), cam_mask=0xFFFFFFFF, settings=SETTINGS):
    fo, ff, oc, fc = cam
    ctx.cull([ff], cam_mask=[cam_mask])
    ctx.cull_shadow_casters(0, np.array(eye, f32), *settings, csm_camera=fc)
    maps, entries = ctx.get_shadow_maps()
    want = co.shadow_maps(og, sc.flags, fo, eye, cam_mask, settings, sc.sources, sc.scale(), csm=oc)
    assert [(int(m["light"]), int(m["face"]), int(m["cascade"])) for m in maps] == [(w[0], w[1], w[2]) for w in want]
    for m, w in zip(maps, want):
        assert same_bits(m["view_projection"], w[3]), (int(m["light"]), int(m["face"]), int(m["cascade"]))
        got = np.sort(entries[m["first"]: m["first"] + m["count"]])
        assert np.array_equal(got, w[4]), (int(m["light"]), int(m["cascade"]), len(got), len(w[4]))
    return maps, entries


def n_cascades(maps, sc):
    return sum(1 for m in maps if sc.sources[int(m["light"])][0] == DIR)


@pytest.mark.parametrize("relative", [0, 1])
@pytest.mark.parametrize("kind", [co.PERSPECTIVE, co.ORTHOGRAPHIC])
@pytest.mark.parametrize("seed", [0, 1])
def test_random_scenes_match_the_oracle(ctx, seed, kind, relative):
    rng = np.random.default_rng(1700 + 10 * seed + 2 * kind + relative)
    sc = ShadowScene(rng, 4000, 40)
    og = sc.load(ctx)
    cam = camera(kind, size=25.0)
    dirs = [n for n in sc.lights.tolist() if sc.sources[n][0] == DIR]
    opts = random_options(rng, dirs[1:], relative)  # the first directional light keeps the default options
    if len(dirs) > 2 and not relative:
        opts[dirs[2]] = (0, (0.1, 0.1, 30.0))  # a split equal to z_near: MIN_DEPTH_DELTA, and a collapsed second cascade
    send_options(ctx, cam[2], opts)
    maps, _ = compare(ctx, og, sc, cam)
    assert n_cascades(maps, sc) >= 3 and len(maps) > n_cascades(maps, sc)
    # another camera: moved and turned, a mask that drops some nodes, different settings
    cam2 = camera(kind, eye=(3.0, 1.0, -10.0), target=(2.0, 0.5, -11.0), z_near=0.5, z_far=90.0, frame=(800.0, 600.0), size=12.0)
    cam2[2].options = cam[2].options
    compare(ctx, og, sc, cam2, eye=(3.0, 1.0, -10.0), cam_mask=0x1, settings=(25.0, 60.0, 1, 0))


def test_odd_cameras_match_the_oracle(ctx):
    """z_far < z_near (the swap), tiny and negative vertical sizes, a frame with h = 0 and a frame with w = h = 0."""
    rng = np.random.default_rng(1750)
    sc = ShadowScene(rng, 1500, 16, kinds=(DIR, 2))
    og = sc.load(ctx)
    for kind, kw in ((co.PERSPECTIVE, dict(z_near=150.0, z_far=0.1)), (co.ORTHOGRAPHIC, dict(size=1e-7)), (co.ORTHOGRAPHIC, dict(size=-8.0)),
                     (co.ORTHOGRAPHIC, dict(size=-1e-7)), (co.PERSPECTIVE, dict(frame=(640.0, 0.0))), (co.ORTHOGRAPHIC, dict(size=5.0, frame=(0.0, 0.0)))):
        cam = camera(kind, **kw)
        send_options(ctx, cam[2], {int(sc.lights[0]): (1, (0.1, 0.5, 1.0))})
        compare(ctx, og, sc, cam)


def test_disabled_and_null_camera_give_the_spot_and_point_maps(ctx):
    rng = np.random.default_rng(1760)
    sc = ShadowScene(rng, 3000, 30)
    og = sc.load(ctx)
    assert any(sc.sources[n][0] == DIR for n in sc.lights.tolist())
    fo, ff, oc, fc = camera(enabled=False)
    ctx.cull([ff])
    ctx.cull_shadow_casters(0, np.zeros(3, f32), *SETTINGS)
    m0, e0 = ctx.get_shadow_maps()
    ctx.cull_shadow_casters(0, np.zeros(3, f32), *SETTINGS, csm_camera=fc)
    m1, e1 = ctx.get_shadow_maps()
    assert m0.tobytes() == m1.tobytes()  # the same table and list places; the order inside a list is unspecified
    for m in m1:
        sl = slice(int(m["first"]), int(m["first"] + m["count"]))
        assert np.array_equal(np.sort(e0[sl]), np.sort(e1[sl]))
    want = so.shadow_maps(og, sc.flags, fo, (0.0, 0.0, 0.0), 0xFFFFFFFF, SETTINGS, sc.sources, sc.scale())
    assert [(int(m["light"]), int(m["face"])) for m in m1] == [(w[0], w[1]) for w in want]
    assert len(co.shadow_maps(og, sc.flags, fo, (0.0, 0.0, 0.0), 0xFFFFFFFF, SETTINGS, sc.sources, sc.scale(), csm=oc)) == len(want)
    # enabled again: the cascades appear between the other maps
    cam = camera()
    maps, _ = compare(ctx, og, sc, cam)
    assert n_cascades(maps, sc) > 0


def test_gates_and_zero_scale(ctx):
    rng = np.random.default_rng(1770)
    sc = ShadowScene(rng, 2000, 8, kinds=(DIR,), p_cast=1.0)
    in_view(rng, sc)
    og = sc.load(ctx)
    cam = camera()
    maps, _ = compare(ctx, og, sc, cam)
    assert len(maps) == 3 * len(sc.lights)
    # no cast_shadows on one light, a zero scale on another (max(scale) * f32::MAX = 0: the sphere test decides)
    a, b = int(sc.lights[0]), int(sc.lights[1])
    sc.flags[a] &= ~np.uint32(fb.NODE_CAST_SHADOWS)
    ctx.set_flags(sc.flags[a:a + 1], np.array([a], np.uint32))
    og.L.orc_node_set_cast_shadows(og.h, a, 0)
    sc.trs[b, 7:10] = 0.0
    ctx.set_local_trs(sc.trs[b:b + 1], np.array([b], np.uint32))
    og.set_local_matrix(b, local_from_trs(sc.trs[b:b + 1])[0])
    og.update()
    ctx.update_transforms(fb.UPDATE_ALL)
    maps, _ = compare(ctx, og, sc, cam)
    assert a not in maps["light"].tolist()


def rotation_animation(rng, sc, nodes):
    keys, tracks = [], []
    for node in nodes:
        t = np.zeros((), ob.TRACK_DTYPE)
        t["target_node"], t["binding"], t["value_kind"], t["enabled"], t["n_curves"] = node, ob.BIND_ROTATION, ob.TV_QUAT_EULER, 1, 3
        for c in range(3):
            t["first_key"][c], t["n_keys"][c] = len(keys), 2
            keys.append((0.0, float(rng.uniform(-1.5, 1.5)), 1, 0.0, 0.0))
            keys.append((2.0, float(rng.uniform(-1.5, 1.5)), 1, 0.0, 0.0))
        tracks.append(t)
    kk = np.zeros(len(keys), ob.KEY_DTYPE)
    for i, k in enumerate(keys):
        kk[i] = k
    return np.array(tracks, ob.TRACK_DTYPE), kk


def test_suns_rotated_between_frames_by_trs_and_animate(ctx):
    rng = np.random.default_rng(1781)
    sc = ShadowScene(rng, 2000, 12, kinds=(DIR, 1, 2))
    og = sc.load(ctx)
    cam = camera()
    dirs = [n for n in sc.lights.tolist() if sc.sources[n][0] == DIR]
    assert len(dirs) >= 4
    send_options(ctx, cam[2], random_options(rng, dirs[::2], 1))
    before, _ = compare(ctx, og, sc, cam)
    # frame 2: fyx_set_local_trs turns half of the suns
    moved = np.array(dirs[::2], np.uint32)
    sc.trs[moved, 3:7] = rand_quat(rng, len(moved))
    loc = local_from_trs(sc.trs[moved])
    for i, node in enumerate(moved.tolist()):
        og.set_local_matrix(node, loc[i])
    og.update()
    ctx.set_local_trs(sc.trs[moved], moved)
    ctx.update_transforms(fb.UPDATE_INCREMENTAL)
    after, _ = compare(ctx, og, sc, cam)
    turned = [m["view_projection"].tobytes() for m in after if int(m["light"]) in moved.tolist()]
    assert turned and set(turned).isdisjoint(m["view_projection"].tobytes() for m in before)
    # frames 3..: fyx_animate turns the other suns
    animated = dirs[1::2]
    tk, kk = rotation_animation(rng, sc, animated)
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
    for _ in range(3):
        ob.update_animations([anim], 0.375, og, arr)
        og.update()
        ctx.animate(0.375)
        ctx.update_transforms(fb.UPDATE_INCREMENTAL)
        compare(ctx, og, sc, cam)


def test_fyx_cull_with_the_cascade_matrices_gives_the_same_sets(ctx):
    rng = np.random.default_rng(1790)
    sc = ShadowScene(rng, 5000, 20, kinds=(DIR, 2))
    og = sc.load(ctx)
    cam = camera(co.ORTHOGRAPHIC, size=30.0)
    send_options(ctx, cam[2], {})
    maps, entries = compare(ctx, og, sc, cam)
    casc = [k for k, m in enumerate(maps) if sc.sources[int(m["light"])][0] == DIR]
    assert len(casc) >= 6
    for b in range(0, len(casc), 8):
        chunk = casc[b: b + 8]
        frusta = [fb.frustum_from_view_projection_matrix(maps[k]["view_projection"].copy()) or fb.frustum_default() for k in chunk]
        ctx.cull(frusta, cam_mask=[0xFFFFFFFF] * len(frusta), pass_flags=[fb.PASS_SHADOW] * len(frusta))
        for j, k in enumerate(chunk):
            m = maps[k]
            assert np.array_equal(np.sort(ctx.get_visible(j)), np.sort(entries[m["first"]: m["first"] + m["count"]]))


def test_pack_shadow_instances_over_cascades(ctx):
    """Cascade instances are sorted by the map's look_at_lh; skinned surfaces with their bone blocks included."""
    rng = np.random.default_rng(1800)
    sc = ShadowScene(rng, 3000, 10, spread=12.0, depth_z=(-30.0, -2.0), kinds=(DIR, 1, 2), p_cast=1.0)
    in_view(rng, sc)
    og = sc.load(ctx)
    bundle = with_bundles(ctx, rng, sc.n)
    renderable = np.flatnonzero((sc.flags & fb.NODE_RENDERABLE) != 0)
    meshes = rng.choice(renderable[renderable > 0], 60, replace=False)
    bone_ib, surfaces = {}, []
    for mesh in meshes.tolist():
        bones = rng.choice(np.arange(1, sc.n), int(rng.integers(1, 9)), replace=False).astype(np.uint32)
        for b in bones.tolist():
            if b not in bone_ib:
                ib = np.eye(4, dtype=f32)
                ib[3, 0:3] = rng.uniform(-2, 2, 3)
                bone_ib[b] = ib.reshape(16)
                og.set_inv_bind(b, bone_ib[b])
        og.add_surface(mesh, bones)
        sid = ctx.add_skinned_surface(mesh, bones, np.stack([bone_ib[b] for b in bones.tolist()]), None, n_verts=0)
        surfaces.append([(int(bundle[mesh]), sid)])
    ctx.set_node_surfaces(meshes.tolist(), surfaces)
    multi = {int(n): 1 for n in meshes.tolist()}
    og.update_hierarchical_data()
    ctx.update_transforms(fb.UPDATE_ALL)
    ctx.build_palettes()
    cam = camera()
    send_options(ctx, cam[2], random_options(rng, sc.lights.tolist(), 0))
    fo, ff, oc, fc = cam
    ctx.enable_instances()
    maps, entries = compare(ctx, og, sc, cam, settings=(200.0, 200.0, 1, 1))
    ctx.pack_shadow_instances()
    ctx.pack_shadow_bone_matrices()
    want = co.shadow_maps(og, sc.flags, fo, (0.0, 0.0, 0.0), 0xFFFFFFFF, (200.0, 200.0, 1, 1), sc.sources, sc.scale(), csm=oc)
    views = {}
    n_casc = n_blocks = 0
    for k, (m, w) in enumerate(zip(maps, want)):
        light = int(m["light"])
        if sc.sources[light][0] == DIR:
            if light not in views:
                views[light] = co.cascade_views(og, light, oc)
            view = views[light][int(m["cascade"])]
            n_casc += 1
        else:
            view = map_view(og, sc.sources, light, int(m["face"]))
        check_map(ctx, og, k, m, entries, w + (view,), lambda n, s: int(bundle[n]), multi=multi)
        inst = ctx.get_shadow_instances(k)
        for i in range(inst["node"].size):
            nd, sf = int(inst["node"][i]), int(inst["surface"][i])
            blk = ctx.get_shadow_bone_matrix_block(k, i)
            want_blk = np.empty(255 * 16, f32)
            if nd in multi:
                has = ob.lib().orc_surface_bone_block(og.h, nd, sf, ob.fp(want_blk))
            else:
                has = ob.lib().orc_instance_bone_block(og.h, nd, ob.fp(want_blk))
            assert bool(has) == (blk is not None)
            if has:
                assert blk.reshape(-1).tobytes() == want_blk.tobytes()
                n_blocks += sc.sources[light][0] == DIR
    assert n_casc >= 6 and n_blocks > 10


def test_one_million_nodes_four_suns_and_point_lights_compared_in_full(ctx):
    rng = np.random.default_rng(1810)
    sc = ShadowScene(rng, 1_000_000, 12, spread=40.0, rotate_all=False, kinds=(2,), p_cast=1.0)
    in_view(rng, sc)
    for k, node in enumerate(sc.lights.tolist()):
        sc.sources[node] = (DIR, f32(0.0), f32(0.0)) if k < 4 else (fb.LIGHT_POINT, f32(0.0), f32(rng.uniform(4.0, 12.0)))
    og = sc.load(ctx)
    cam = camera()
    send_options(ctx, cam[2], random_options(rng, sc.lights[:2].tolist(), 1))
    maps, entries = compare(ctx, og, sc, cam, settings=(200.0, 200.0, 1, 1))
    assert n_cascades(maps, sc) == 12 and len(maps) >= 12 + 6 and len(entries) > 100_000


def code_of(fn):
    with pytest.raises(fb.FyxError) as e:
        fn()
    return e.value.code


def test_errors(ctx):
    rng = np.random.default_rng(1820)
    sc = ShadowScene(rng, 500, 6)
    og = sc.load(ctx)
    t = np.zeros(3, f32)
    fo, ff, oc, fc = camera()
    assert code_of(lambda: ctx.cull_shadow_casters(0, t, csm_camera=fc)) == L.FYX_ERR_STATE  # no cull yet
    ctx.cull([ff])
    assert code_of(lambda: ctx.cull_shadow_casters(1, t, csm_camera=fc)) == L.FYX_ERR_INVALID_ARGUMENT
    bad = camera()[3]
    bad.projection = 7
    assert code_of(lambda: ctx.cull_shadow_casters(0, t, csm_camera=bad)) == L.FYX_ERR_INVALID_ARGUMENT
    ctx.cull_shadow_casters(0, t, csm_camera=fc)
    ctx.render_prep(frusta=[ff], async_=True, readback_visible=True, do_palettes=False, do_skin=False)
    assert code_of(lambda: ctx.cull_shadow_casters(0, t, csm_camera=fc)) == L.FYX_ERR_STATE  # a frame in flight
    ctx.frame_wait()
    ctx.cull_shadow_casters(0, t, csm_camera=fc)
    # the options call
    opt = np.zeros(1, fb.Context.CSM_OPTIONS_DTYPE)
    assert code_of(lambda: ctx.set_csm_options(opt, np.array([sc.n], np.uint32))) == L.FYX_ERR_INVALID_ARGUMENT
    opt["relative"] = 2
    assert code_of(lambda: ctx.set_csm_options(opt, np.array([1], np.uint32))) == L.FYX_ERR_INVALID_ARGUMENT
    # LOD ranges with observers, then a static batch: refused as by fyx_cull_shadow_casters
    ctx.set_lod_ranges(np.array([0.0, 0.5], f32), np.array([int(sc.lights[0])], np.uint32))
    ctx.set_observers([((0, 0, 0), 0.1, 150.0)])
    ctx.cull([ff])
    assert code_of(lambda: ctx.cull_shadow_casters(0, t, csm_camera=fc)) == L.FYX_ERR_STATE
    ctx.set_observers([])
    flags = sc.flags.copy()
    flags[5] |= fb.NODE_STATIC_BATCH
    ctx.set_flags(flags[5:6], np.array([5], np.uint32))
    ctx.update_transforms(fb.UPDATE_ALL)
    ctx.cull([ff])
    assert code_of(lambda: ctx.cull_shadow_casters(0, t, csm_camera=fc)) == L.FYX_ERR_STATE
    del og
