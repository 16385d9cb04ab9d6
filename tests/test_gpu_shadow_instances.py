"""N3 for the shadow maps: fyx_pack_shadow_instances packs every map of the last fyx_cull_shadow_casters as fyx_pack_instances
packs a frustum, for the map's observer (view_matrix = its look_at_rh, view_projection = its matrix).

Per map, against the oracle (tests/shadow_oracle.py for the maps, the C oracle's from_graph / collect_render_data for the
instances): the node set, sort index / world / wvp bit for bit, the bundle table as a partition with ascending ids and the
sort index of the first-pushed instance; meshes with several surfaces and skinned surfaces with their bone blocks; and at
scale, bit for bit the same as fyx_pack_instances after fyx_cull of the map frusta."""
import ctypes as C

import numpy as np
import pytest

import fyrox_b200 as fb
import oracle_binding as ob
import shadow_oracle as so
from fyrox_b200 import _lib as L
from helpers import camera_frustum, preorder_rank
from test_gpu_shadow_casters import ShadowScene, in_view

pytestmark = pytest.mark.gpu

f32 = np.float32
SETTINGS = (40.0, 40.0, 1, 1)
BIG = (200.0, 200.0, 1, 1)


def map_view(og, sources, light, face):
    """The view matrix of a shadow map, the observer's view_matrix of its shadow pass: the look_at_rh that
    shadow_oracle.shadow_maps multiplies into the map's view_projection (spot: light.rs:706-722; point: shadow/point.rs:172-180)."""
    g = og.global_transform(light)
    position = g[12:15].astype(f32)
    if sources[light][0] == so.LIGHT_SPOT:
        emit_direction = so.try_normalize(g[4:7].astype(f32), so.F32_EPSILON, (0.0, 0.0, 1.0))
        up = so.try_normalize(g[8:11].astype(f32), so.F32_EPSILON, (0.0, 1.0, 0.0))
        return ob.look_at_rh(position, position - emit_direction, up)
    look, up = so.CUBE_FACES[face]
    return ob.look_at_rh(position, position + np.array(look, f32), np.array(up, f32))


def shadow_cull(ctx, og, sc, settings=SETTINGS, cam_mask=0xFFFFFFFF):
    """Camera cull, shadow cull with instances enabled, pack; returns the oracle's maps, each with its view matrix."""
    fo, ff = camera_frustum((0.0, 0.0, 0.0), (0.0, 0.0, -1.0), zfar=150.0)
    ctx.enable_instances()
    ctx.cull([ff], cam_mask=[cam_mask])
    ctx.cull_shadow_casters(0, np.zeros(3, f32), *settings)
    ctx.pack_shadow_instances()
    want = [w + (map_view(og, sc.sources, w[0], w[1]),)
            for w in so.shadow_maps(og, sc.flags, fo, (0.0, 0.0, 0.0), cam_mask, settings, sc.sources, sc.scale())]
    maps, entries = ctx.get_shadow_maps()
    assert [(int(m["light"]), int(m["face"])) for m in maps] == [(w[0], w[1]) for w in want]
    return maps, entries, want


def check_map(ctx, og, k, m, entries, w, key_of, rank=False, cam_mask=0xFFFFFFFF, per_instance=True, multi=None):
    """Map k's instances against the oracle.  key_of(node, surface) = the bundle id; multi = {node: n_surfaces} for nodes
    given several surfaces (they are checked per surface by orc_node_surface_instance)."""
    multi = multi or {}
    _, _, _, vp, vis, view = w
    inst = ctx.get_shadow_instances(k)
    node, surf = inst["node"], inst["surface"]
    listed = np.sort(entries[m["first"]: m["first"] + m["count"]])
    assert np.array_equal(listed, vis)
    # one instance per (listed node, surface)
    pairs = sorted(zip(node.tolist(), surf.tolist()))
    assert pairs == sorted((int(n), s) for n in vis for s in range(multi.get(int(n), 1)))
    if per_instance:
        for i in range(node.size):
            nd, sf = int(node[i]), int(surf[i])
            if nd in multi:
                ww, wvp = np.empty(16, f32), np.empty(16, f32)
                sk = C.c_int()
                si = ob.lib().orc_node_surface_instance(og.h, nd, sf, ob.fp(np.ascontiguousarray(view)), ob.fp(np.ascontiguousarray(vp)), ob.fp(ww),
                                                        ob.fp(wvp), C.byref(sk))
            else:
                si, ww, wvp = og.instance(nd, view, vp)
            assert int(inst["sort_index"][i]) == si, (k, nd, sf)
            assert inst["world"][i].tobytes() == ww.tobytes() and inst["wvp"][i].tobytes() == wvp.tobytes(), (k, nd, sf)
    # bundle table: ascending non-empty ids, a partition of the map's instances, each instance in its key's bundle
    b = inst["bundles"]
    keys = np.array([key_of(int(n), int(s)) for n, s in zip(node, surf)], np.int64)
    assert np.array_equal(b["id"], np.unique(keys))
    assert int(b["count"].sum()) == node.size
    assert np.array_equal(b["first"], np.concatenate([[0], np.cumsum(b["count"])[:-1]]).astype(np.uint32)) if b.size else node.size == 0
    # sort index of the bundle = that of the instance pushed first: the DFS order of the map's from_graph, else the lowest node
    fr = ob.frustum_from_vp(vp) or so.default_frustum()
    dfs = og.from_graph(fr, cam_mask, shadow_pass=True)
    first_pushed = {}
    for n_ in dfs.tolist():
        for s in range(multi.get(n_, 1)):
            first_pushed.setdefault(key_of(n_, s), n_)
    for row in b:
        sl = slice(int(row["first"]), int(row["first"] + row["count"]))
        assert (keys[sl] == row["id"]).all()
        lead = first_pushed[int(row["id"])] if rank else int(node[sl].min())
        assert int(row["sort_index"]) == og.instance(lead, view, vp)[0]
    return node.size


def with_bundles(ctx, rng, n, hi=41):
    bundle = rng.integers(0, hi, n).astype(np.uint32)
    bundle[bundle % 7 == 3] += 1  # holes in the id space
    ctx.set_bundle_ids(bundle)
    return bundle


@pytest.mark.parametrize("seed", [0, 2])
def test_every_map_matches_the_oracle_with_and_without_dfs_order(ctx, seed):
    rng = np.random.default_rng(700 + seed)  # the scenes of test_gpu_shadow_casters.test_random_scenes_match_the_oracle
    sc = ShadowScene(rng, 4000, 40)
    og = sc.load(ctx)
    bundle = with_bundles(ctx, rng, sc.n)
    maps, entries, want = shadow_cull(ctx, og, sc)
    assert len(maps) > 0
    total = sum(check_map(ctx, og, k, maps[k], entries, want[k], lambda n, s: int(bundle[n])) for k in range(len(maps)))
    assert total > 100
    # the DFS order decides each bundle's sort index
    ctx.set_dfs_order(preorder_rank(sc.parent))
    maps, entries, want = shadow_cull(ctx, og, sc, cam_mask=0x3)
    for k in range(len(maps)):
        check_map(ctx, og, k, maps[k], entries, want[k], lambda n, s: int(bundle[n]), rank=True, cam_mask=0x3)


def test_meshes_with_several_surfaces_and_skinned_surfaces(ctx):
    rng = np.random.default_rng(931)
    sc = ShadowScene(rng, 3000, 16, spread=12.0, depth_z=(-30.0, -2.0), kinds=(1, 2), p_cast=1.0)
    in_view(rng, sc)
    og = sc.load(ctx)
    bundle = with_bundles(ctx, rng, sc.n)
    # palette-only skinned surfaces on some renderable nodes, bones elsewhere in the graph
    renderable = np.flatnonzero((sc.flags & fb.NODE_RENDERABLE) != 0)
    meshes = rng.choice(renderable[renderable > 0], 120, replace=False)
    nodes, surfaces, want_key = [], [], {}
    bone_ib = {}
    for i, mesh in enumerate(meshes.tolist()):
        lst = []
        n_surf = int(rng.integers(1, 4))
        for s in range(n_surf):
            bid = int(rng.integers(50, 60))
            if i % 3 != 2 and s != 1:  # skinned
                bones = rng.choice(np.arange(1, sc.n), int(rng.integers(1, 9)), replace=False).astype(np.uint32)
                for b in bones.tolist():
                    if b not in bone_ib:
                        ib = np.eye(4, dtype=f32)
                        ib[3, 0:3] = rng.uniform(-2, 2, 3)
                        bone_ib[b] = ib.reshape(16)
                        og.set_inv_bind(b, bone_ib[b])
                og.add_surface(mesh, bones)
                sid = ctx.add_skinned_surface(mesh, bones, np.stack([bone_ib[b] for b in bones.tolist()]), None, n_verts=0)
            else:
                og.add_surface(mesh, np.empty(0, np.uint32))
                sid = None
            lst.append((bid, sid))
            want_key[(mesh, s)] = bid
        nodes.append(mesh)
        surfaces.append(lst)
    ctx.set_node_surfaces(nodes, surfaces)
    og.update_hierarchical_data()
    ctx.update_transforms(fb.UPDATE_ALL)
    ctx.build_palettes()
    multi = {n_: len(l) for n_, l in zip(nodes, surfaces)}
    key_of = lambda n, s: want_key.get((n, s), int(bundle[n]))  # noqa: E731
    maps, entries, want = shadow_cull(ctx, og, sc, settings=BIG)
    ctx.pack_shadow_bone_matrices()
    n_multi = n_blocks = n_plain = 0
    for k in range(len(maps)):
        check_map(ctx, og, k, maps[k], entries, want[k], key_of, multi=multi)
        inst = ctx.get_shadow_instances(k)
        for i in range(inst["node"].size):
            nd, sf = int(inst["node"][i]), int(inst["surface"][i])
            blk = ctx.get_shadow_bone_matrix_block(k, i)
            want_blk = np.empty(255 * 16, f32)
            if nd in multi:
                has = ob.lib().orc_surface_bone_block(og.h, nd, sf, ob.fp(want_blk))
            else:
                has = ob.lib().orc_instance_bone_block(og.h, nd, ob.fp(want_blk))
            assert bool(has) == (blk is not None), (k, nd, sf)
            if has:
                assert blk.reshape(-1).tobytes() == want_blk.tobytes()
                assert inst["world"][i].tobytes() == np.eye(4, dtype=f32).reshape(16).tobytes()
                n_blocks += 1
            else:
                n_plain += 1
            n_multi += nd in multi
    assert n_multi > 30 and n_blocks > 10 and n_plain > 100


def test_zero_maps_empty_lists_many_maps_and_several_groups(ctx):
    rng = np.random.default_rng(932)
    # > 256 maps
    sc = ShadowScene(rng, 3000, 60, spread=12.0, depth_z=(-30.0, -2.0), kinds=(2,), p_cast=1.0)
    in_view(rng, sc)
    og = sc.load(ctx)
    bundle = with_bundles(ctx, rng, sc.n)
    maps, entries, want = shadow_cull(ctx, og, sc, settings=BIG)
    assert len(maps) > 256
    for k in range(len(maps)):
        check_map(ctx, og, k, maps[k], entries, want[k], lambda n, s: int(bundle[n]), per_instance=k % 16 == 0)
    # more bins than one group holds: bundle id 2^24 - 1 and three lights (18 maps, two per group)
    hot = int(entries[0])  # a node some map lists
    big = bundle.copy()
    big[hot] = (1 << 24) - 1
    ctx.set_bundle_ids(big[hot:hot + 1], np.array([hot], np.uint32))
    keep = sorted(sc.sources)[:3]
    ShadowScene.send_sources(ctx, {k: (fb.LIGHT_UNKNOWN, 0.0, 0.0) for k in sorted(sc.sources)[3:]})
    sc.sources = {k: sc.sources[k] for k in keep}
    maps, entries, want = shadow_cull(ctx, og, sc, settings=BIG)
    assert len(maps) == 18
    for k in range(len(maps)):
        check_map(ctx, og, k, maps[k], entries, want[k], lambda n, s: int(big[n]), per_instance=k % 4 == 0)
    assert any(hot in entries[m["first"]: m["first"] + m["count"]] for m in maps)
    # maps with empty lists among full ones: a scene where almost nothing casts shadows and the lights are not meshes
    sc = ShadowScene(rng, 3000, 12, spread=12.0, depth_z=(-30.0, -2.0), kinds=(1, 2), p_cast=0.004)
    in_view(rng, sc)
    sc.flags[sc.lights] &= ~np.uint32(fb.NODE_RENDERABLE)
    og = sc.load(ctx)
    bundle = with_bundles(ctx, rng, sc.n)
    maps, entries, want = shadow_cull(ctx, og, sc, settings=BIG)
    counts = [int(m["count"]) for m in maps]
    assert 0 in counts and max(counts) > 0
    for k in range(len(maps)):
        check_map(ctx, og, k, maps[k], entries, want[k], lambda n, s: int(bundle[n]))
    # zero maps
    ShadowScene.send_sources(ctx, {k: (fb.LIGHT_UNKNOWN, 0.0, 0.0) for k in sc.sources})
    sc.sources = {}
    maps, entries, want = shadow_cull(ctx, og, sc, settings=BIG)
    assert len(maps) == 0
    assert code_of(lambda: ctx.get_shadow_instances(0)) == L.FYX_ERR_INVALID_ARGUMENT


def test_one_million_nodes_forty_maps_equal_fyx_pack_instances(ctx):
    rng = np.random.default_rng(933)
    sc = ShadowScene(rng, 1_000_000, 20, spread=40.0, rotate_all=False, kinds=(1, 2), p_cast=1.0)
    in_view(rng, sc)
    for node in sc.lights.tolist():
        sc.sources[node] = (fb.LIGHT_POINT if node % 3 else fb.LIGHT_SPOT, f32(1.2), f32(rng.uniform(4.0, 12.0)))
    og = sc.load(ctx)
    with_bundles(ctx, rng, sc.n, hi=300)
    ctx.set_dfs_order(preorder_rank(sc.parent))
    maps, entries, want = shadow_cull(ctx, og, sc, settings=BIG)
    assert len(maps) >= 40 and len(entries) > 100_000
    got = [ctx.get_shadow_instances(k) for k in range(len(maps))]
    for b in range(0, len(maps), 8):
        chunk = maps[b: b + 8]
        frusta = [fb.frustum_from_view_projection_matrix(m["view_projection"]) or fb.frustum_default() for m in chunk]
        ctx.cull(frusta, pass_flags=[fb.PASS_SHADOW] * len(frusta))
        for k, m in enumerate(chunk):
            ref = ctx.pack_instances(k, want[b + k][5], m["view_projection"])
            g = got[b + k]
            assert g["node"].size == ref["node"].size > 0
            assert g["bundles"].tobytes() == ref["bundles"].tobytes(), b + k
            # the order inside a bundle is unspecified: compare per (node, surface)
            og_, ow = np.lexsort((g["surface"], g["node"])), np.lexsort((ref["surface"], ref["node"]))
            for key in ("node", "surface", "sort_index", "world", "wvp"):
                assert g[key][og_].tobytes() == ref[key][ow].tobytes(), (b + k, key)


def test_state_and_argument_errors(ctx):
    rng = np.random.default_rng(934)
    sc = ShadowScene(rng, 600, 8, spread=12.0, depth_z=(-30.0, -2.0), kinds=(1, 2), p_cast=1.0)
    in_view(rng, sc)
    og = sc.load(ctx)
    t = np.zeros(3, f32)
    _, ff = camera_frustum(zfar=150.0)
    assert code_of(lambda: ctx.pack_shadow_instances()) == L.FYX_ERR_STATE  # no shadow cull
    ctx.cull([ff])
    ctx.cull_shadow_casters(0, t, *BIG)
    assert code_of(lambda: ctx.pack_shadow_instances()) == L.FYX_ERR_STATE  # made without enable_instances
    ctx.enable_instances()
    assert code_of(lambda: ctx.pack_shadow_bone_matrices()) == L.FYX_ERR_STATE  # no pack yet
    ctx.cull([ff])
    ctx.cull_shadow_casters(0, t, *BIG)
    ctx.pack_shadow_instances()
    n_maps = len(ctx.get_shadow_maps()[0])
    assert n_maps > 0
    assert code_of(lambda: ctx.get_shadow_instances(n_maps)) == L.FYX_ERR_INVALID_ARGUMENT
    assert code_of(lambda: ctx.get_shadow_bone_matrix_block(0, 0)) == L.FYX_ERR_STATE  # blocks not packed
    ctx.pack_shadow_bone_matrices()
    assert code_of(lambda: ctx.get_shadow_bone_matrix_block(n_maps, 0)) == L.FYX_ERR_INVALID_ARGUMENT
    # a frame in flight
    ctx.render_prep(frusta=[ff], async_=True, readback_visible=True, do_palettes=False, do_skin=False)
    assert code_of(lambda: ctx.pack_shadow_instances()) == L.FYX_ERR_STATE
    ctx.frame_wait()
    ctx.cull([ff])
    ctx.cull_shadow_casters(0, t, *BIG)
    ctx.pack_shadow_instances()
    # a topology change makes the recorded slots stale
    ctx.set_topology(sc.parent, sc.flags, sc.mask, sc.aabb)
    assert code_of(lambda: ctx.pack_shadow_instances()) == L.FYX_ERR_STATE
    # a new shadow cull drops the packed result
    sc.load(ctx)
    ctx.cull([ff])
    ctx.cull_shadow_casters(0, t, *BIG)
    assert code_of(lambda: ctx.get_shadow_instances(0)) == L.FYX_ERR_STATE
    ctx.pack_shadow_instances()
    ctx.get_shadow_instances(0)
    del og


def code_of(fn):
    with pytest.raises(fb.FyxError) as e:
        fn()
    return e.value.code
