"""Sprites and 2D rectangles on the device (fyx_set_sprites): each pack's dynamic batches, quads and Dynamic meshes together,
against tests/dynamic_batch_oracle.py run over the same pass in DFS order, byte for byte; the gates by pass kind; quad nodes are
never ordinary instances; records follow their nodes; set-then-clear launches and returns what a context that never set
quads does; the refusals leave the state as it was; the scene mirror end to end."""
import ctypes as C

import numpy as np
import pytest

import dynamic_batch_oracle as dbo
import sprite_batch_oracle as sbo
import fyrox_b200 as fb
from fyrox_b200.context import Context
from helpers import camera_frustum, preorder_rank
from test_gpu_dynamic_batches import EYE, assert_same, canonical, expect, push_order, register
from test_gpu_instance_pack import launches
from test_gpu_shadow_casters import ShadowScene, in_view
from test_gpu_shadow_instances import shadow_cull

pytestmark = pytest.mark.gpu

f32 = np.float32
NONE = dbo.NONE
SPRITE_L, RECT_L = 2, 3  # layout ids; register() uses 0 and 1 with batch keys 0..5
SPRITE_LAYOUT = (40, 0, NONE, NONE)
RECT_LAYOUT = (24, 0, NONE, NONE)
SPRITE_KEYS, RECT_KEYS = (10, 11), (20, 21)


def random_quad(rng, kind):
    keys, lid = (SPRITE_KEYS, SPRITE_L) if kind == sbo.SPRITE else (RECT_KEYS, RECT_L)
    return sbo.Quad(kind, int(rng.choice(keys)), lid, tuple(rng.uniform(-1, 1, 4).astype(f32).tolist()),
                    tuple(int(x) for x in rng.integers(0, 256, 4)), float(rng.uniform(-2, 2)), float(rng.uniform(-3, 3)),
                    bool(rng.random() < 0.5), bool(rng.random() < 0.5))


def set_quads(ctx, quads):
    nodes = sorted(quads)
    ctx.set_sprites(np.array(nodes, np.uint32), np.array([quads[n].record() for n in nodes], Context.SPRITE))


def add_quads(ctx, rng, sc, n_surf, dyn, p=0.5, exclude=(), sprite_meshes=40):
    """Quads on about `p` of the renderable nodes that have no surfaces (not the lights), plus `sprite_meshes` Dynamic meshes
    with the SpriteVertex or the RectangleVertex layout, in turn, under the quads' keys (3 to 9 vertices: the quads after an odd
    count start at an odd vertex, which takes the 8-byte stores)."""
    free = np.flatnonzero((sc.flags & fb.NODE_RENDERABLE) != 0)
    free = np.setdiff1d(free[free > 0], np.concatenate([np.array(list(n_surf), np.int64), sc.lights.astype(np.int64),
                                                         np.asarray(exclude, np.int64)]))
    pick = rng.permutation(free)[: int(len(free) * p)]
    meshes, nodes = pick[:sprite_meshes].tolist(), pick[sprite_meshes:].tolist()
    for j, m in enumerate(meshes):
        keys, lid, layout = (SPRITE_KEYS, SPRITE_L, SPRITE_LAYOUT) if j % 2 == 0 else (RECT_KEYS, RECT_L, RECT_LAYOUT)
        n = int(rng.integers(3, 10))
        raw = rng.integers(0, 256, (n, layout[0]), dtype=np.uint8)
        raw[:, 0:12] = rng.uniform(-3, 3, (n, 3)).astype(f32).view(np.uint8)
        s = dbo.DynSurface(int(rng.choice(keys)), lid, layout, raw.tobytes(),
                           rng.integers(0, n, (int(rng.integers(1, 6)), 3)).astype(np.uint32))
        ctx.add_dynamic_surface(m, 0, s.batch_key, s.layout_id, s.layout, s.vertices, s.triangles)
        dyn[(m, 0)] = s
    quads = {int(n): random_quad(rng, sbo.SPRITE if rng.random() < 0.6 else sbo.RECTANGLE) for n in nodes}
    set_quads(ctx, quads)
    return quads


def build(ctx, seed, n=3000, lights=12, p_cast=0.8, p=0.5):
    rng = np.random.default_rng(seed)
    sc = ShadowScene(rng, n, lights, spread=12.0, depth_z=(-30.0, -2.0), kinds=(1, 2), p_cast=p_cast)
    in_view(rng, sc)
    og = sc.load(ctx)
    ctx.set_bundle_ids(rng.integers(0, 5, sc.n).astype(np.uint32))
    dyn, n_surf = register(ctx, rng, sc, n_meshes=min(300, n // 10))
    quads = add_quads(ctx, rng, sc, n_surf, dyn, p=p)
    ctx.update_transforms(fb.UPDATE_ALL)
    ctx.enable_instances()
    return rng, sc, og, dyn, n_surf, quads


def no_quad_instances(inst, quads):
    assert not set(inst["node"].tolist()) & set(quads)


def check_frustum(ctx, og, sc, dyn, n_surf, quads, rank=None, view=None, shadow=False):
    fo, ff = camera_frustum(zfar=150.0)
    ctx.cull([ff], pass_flags=[fb.PASS_SHADOW if shadow else 0])
    if view is None:
        view = np.eye(4, dtype=f32)
        view[:3, 3] = (0.5, -0.25, 2.0)
        view = view.T.reshape(16).copy()
    inst = ctx.pack_instances(0, view, EYE)
    dfs = [int(n) for n in og.from_graph(fo, shadow_pass=shadow)]
    assert sorted(dfs) == sorted(ctx.get_visible(0).tolist())  # the quad nodes are in the visible list
    want, pushed = expect(og, dfs if rank is not None else sorted(dfs), dyn, n_surf, view, quads=quads, shadow=shadow, flags=sc.flags)
    got = ctx.dynamic_batches("frustum", 0)
    assert_same(got, want, "frustum")
    assert_same(ctx.dynamic_batches("frustum", 0, device=True), want, "frustum device")
    assert sorted(zip(inst["node"].tolist(), inst["surface"].tolist())) == sorted(pushed)
    no_quad_instances(inst, quads)
    return got, set(dfs)


@pytest.mark.parametrize("dfs", [False, True])
def test_camera_frustum_matches_the_oracle(ctx, dfs):
    _, sc, og, dyn, n_surf, quads = build(ctx, 11 + dfs)
    rank = None
    if dfs:
        rank = preorder_rank(sc.parent)
        ctx.set_dfs_order(rank)
    got, vis = check_frustum(ctx, og, sc, dyn, n_surf, quads, rank)
    assert {SPRITE_L, RECT_L} <= set(got["streams"])
    # the cast_shadows quirk is exercised: visible sprites that draw nothing
    assert any(q.kind == sbo.SPRITE and not sc.flags[n] & fb.NODE_CAST_SHADOWS for n, q in quads.items() if n in vis)


def test_shadow_pass_frustum_batches_meshes_only(ctx):
    _, sc, og, dyn, n_surf, quads = build(ctx, 13)
    got, vis = check_frustum(ctx, og, sc, dyn, n_surf, quads, shadow=True)
    assert got["instances"].size > 0 and not set(got["instances"]["node"].tolist()) & set(quads)
    assert vis & set(quads)


def test_every_shadow_map_carries_no_quads(ctx):
    _, sc, og, dyn, n_surf, quads = build(ctx, 14, p_cast=1.0)
    maps, entries, want_maps = shadow_cull(ctx, og, sc)
    assert len(maps) >= 4
    seen = 0
    for k, (m, w) in enumerate(zip(maps, want_maps)):
        nodes = w[4]
        seen += len(set(nodes.tolist()) & set(quads))
        want, pushed = expect(og, push_order(nodes), dyn, n_surf, w[5], quads=quads, shadow=True, flags=sc.flags)
        assert_same(ctx.dynamic_batches("shadow", k), want, ("map", k))
        assert_same(ctx.dynamic_batches("shadow", k, device=True), want, ("map device", k))
        inst = ctx.get_shadow_instances(k)
        assert sorted(zip(inst["node"].tolist(), inst["surface"].tolist())) == sorted(pushed), k
        no_quad_instances(inst, quads)
    assert seen > 50  # the maps' lists do hold quad nodes


def observer_scene(ctx, seed, shadows):
    from test_gpu_observers import ObserverScene
    from test_gpu_scene_shadows import shadowy

    rng = np.random.default_rng(seed)
    s = ObserverScene(rng, 3000, 3, 1)
    if shadows:
        shadowy(s)
    og = s.load(ctx)
    exclude = np.concatenate([s.cam_nodes, s.probe_nodes])
    dyn, n_surf = register(ctx, rng, s.sc, keep_one=shadows, exclude=exclude)
    quads = add_quads(ctx, rng, s.sc, n_surf, dyn, exclude=exclude, sprite_meshes=0 if shadows else 40)
    ctx.update_transforms(fb.UPDATE_ALL)
    ctx.enable_instances()
    return s, og, dyn, n_surf, quads


def test_scene_observers_with_masks_lod_and_static_batches(ctx):
    """Every observer (GBuffer passes, never shadow passes) of a scene with render masks, LOD ranges and static batches."""
    from test_gpu_observers import observe

    s, og, dyn, n_surf, quads = observer_scene(ctx, 21, True)
    table, entries, _, want_obs = observe(ctx, og, s)
    ctx.pack_scene_observer_instances()
    total = 0
    for o, (r, w) in enumerate(zip(table, want_obs)):
        want, pushed = expect(og, push_order(w["visible"]), dyn, n_surf, np.asarray(w["view"], f32).reshape(16), quads=quads,
                              flags=s.sc.flags)
        assert_same(ctx.dynamic_batches("observer", o), want, ("observer", o))
        assert_same(ctx.dynamic_batches("observer", o, device=True), want, ("observer device", o))
        inst = ctx.get_scene_observer_instances(o)
        assert sorted(zip(inst["node"].tolist(), inst["surface"].tolist())) == sorted(pushed), o
        total += sum(1 for i in want["instances"]["node"].tolist() if i in quads)
    assert total > 20


def test_observers_shadow_maps_carry_no_quads(ctx):
    from test_gpu_observers import observe
    from test_gpu_scene_shadows import WIDE

    s, og, dyn, n_surf, quads = observer_scene(ctx, 22, True)
    observe(ctx, og, s)
    ctx.cull_scene_shadow_casters(*WIDE, csm_enabled=True)
    ctx.pack_shadow_instances()
    maps, entries = ctx.get_shadow_maps()
    assert len(maps) >= 4 and int(maps["cascade"].max()) >= 1
    seen = 0
    for k, m in enumerate(maps):
        inst = ctx.get_shadow_instances(k)
        no_quad_instances(inst, quads)
        sort_of = dict(zip(inst["node"].tolist(), inst["sort_index"].tolist()))
        nodes = entries[m["first"]: m["first"] + m["count"]]
        seen += len(set(nodes.tolist()) & set(quads))
        want, pushed = expect(og, push_order(nodes), dyn, n_surf, None, lambda n: sort_of[n], quads, shadow=True, flags=s.sc.flags)
        assert_same(ctx.dynamic_batches("shadow", k), want, ("map", k))
        assert sorted(zip(inst["node"].tolist(), inst["surface"].tolist())) == sorted(pushed), k
    assert seen > 0


def test_size_does_not_change_culling(ctx):
    """A sprite whose size would reach into the frustum but whose unit box does not is culled; the unit box decides."""
    parent = np.array([NONE, 0, 0], np.uint32)
    flags = np.full(3, fb.NODE_DEFAULT | fb.NODE_RENDERABLE, np.uint32)
    flags[0] = fb.NODE_DEFAULT
    aabb = np.tile(np.array([-0.5, -0.5, -0.5, 0.5, 0.5, 0.5], f32), (3, 1))
    ctx.set_topology(parent, flags, np.full(3, 0xFFFFFFFF, np.uint32), aabb)
    local = np.tile(EYE, (3, 1))
    local[1, 12:15] = (0.0, 0.0, -160.0)  # beyond z_far = 150 by more than the unit box
    local[2, 12:15] = (0.0, 0.0, -5.0)
    ctx.set_local_matrices(local)
    ctx.update_transforms(fb.UPDATE_ALL)
    ctx.enable_instances()
    quads = {1: sbo.Quad(sbo.SPRITE, 0, 0, size=1000.0), 2: sbo.Quad(sbo.SPRITE, 0, 0, size=0.001)}
    set_quads(ctx, quads)
    fo, ff = camera_frustum(zfar=150.0)
    ctx.cull([ff])
    assert ctx.get_visible(0).tolist() == [2]
    ctx.pack_instances(0, EYE, EYE)
    d = ctx.dynamic_batches("frustum", 0)
    assert d["instances"]["node"].tolist() == [2] and d["streams"][0]["vertices"].size == 160


def test_record_updates_kind_changes_and_clears_between_packs(ctx):
    rng, sc, og, dyn, n_surf, quads = build(ctx, 31)
    check_frustum(ctx, og, sc, dyn, n_surf, quads)
    nodes = sorted(quads)
    # appearance only: one scatter of the records, no other launch
    for n in nodes[::2]:
        q = random_quad(rng, quads[n].kind)
        q.batch_key, q.layout_id = quads[n].batch_key, quads[n].layout_id
        quads[n] = q
    upd = {n: quads[n] for n in nodes[::2]}
    assert launches(ctx, lambda: set_quads(ctx, upd)) == 1
    check_frustum(ctx, og, sc, dyn, n_surf, quads)
    # kind and key changes, then some nodes cleared
    for n in nodes[1::3]:
        quads[n] = random_quad(rng, sbo.RECTANGLE if quads[n].kind == sbo.SPRITE else sbo.SPRITE)
    set_quads(ctx, {n: quads[n] for n in nodes[1::3]})
    check_frustum(ctx, og, sc, dyn, n_surf, quads)
    gone = nodes[::5]
    ctx.clear_sprites(np.array(gone, np.uint32))
    for n in gone:
        del quads[n]
    check_frustum(ctx, og, sc, dyn, n_surf, quads)


def test_records_follow_their_nodes_across_topology(ctx):
    import oracle_binding as ob

    _, sc, og, dyn, n_surf, quads = build(ctx, 41)
    leaves = sorted(set(quads) - set(sc.parent.tolist()))
    gone = leaves[: len(leaves) // 3]
    flags = sc.flags.copy()
    flags[gone] &= ~np.uint32(fb.NODE_ALIVE)
    ctx.set_topology(sc.parent, flags, sc.mask, sc.aabb)
    ctx.update_transforms(fb.UPDATE_ALL)
    og2 = ob.Graph.build(sc.parent, flags, sc.mask, sc.local, sc.aabb)
    og2.update_hierarchical_data()
    kept = {n: q for n, q in quads.items() if n not in set(gone)}
    check_frustum(ctx, og2, sc, dyn, n_surf, kept)
    # the removed nodes come back as ordinary renderable nodes: one instance each, no quad
    ctx.set_topology(sc.parent, sc.flags, sc.mask, sc.aabb)
    back = np.array(gone, np.uint32)
    ctx.set_local_matrices(sc.local[back], back)
    ctx.update_transforms(fb.UPDATE_ALL)
    check_frustum(ctx, og, sc, dyn, n_surf, kept)


def test_set_then_clear_launches_and_returns_what_never_set_does(ctx):
    """The three packs' launch counts and outputs equal those of a context that never had a quad node."""
    from test_gpu_observers import ObserverScene, observe

    fo, ff = camera_frustum(zfar=150.0)

    def run(c, add):
        rng = np.random.default_rng(50)
        s = ObserverScene(rng, 3000, 3, 1, pruners=False)  # the single-camera shadow cull takes no static batches
        og = s.load(c)
        c.enable_instances()
        quads = {int(n): random_quad(rng, 1 + int(n) % 2) for n in range(1, 3000, 3)
                 if n not in set(s.cam_nodes.tolist()) | set(s.probe_nodes.tolist()) | set(s.sc.lights.tolist())}
        if add:
            set_quads(c, quads)
        c.cull([ff])
        if add:
            c.pack_instances(0, EYE, EYE)
            assert c.dynamic_batches("frustum", 0)["instances"].size > 0
            c.clear_sprites()
        c.cull_shadow_casters(0, np.zeros(3, f32), 200.0, 200.0, 1, 1)
        n = [launches(c, lambda: c.pack_instances(0, EYE, EYE)), launches(c, c.pack_shadow_instances)]
        n_maps = len(c.get_shadow_maps()[0])
        out = [canonical(c.pack_instances(0, EYE, EYE))] + [canonical(c.get_shadow_instances(k)) for k in range(n_maps)]
        table = observe(c, og, s)[0]
        n.append(launches(c, c.pack_scene_observer_instances))
        out += [canonical(c.get_scene_observer_instances(o)) for o in range(len(table))]
        empty = [c.dynamic_batches("frustum", 0)] + [c.dynamic_batches("observer", o) for o in range(len(table))]
        assert all(e["bundles"].size == 0 and not e["streams"] for e in empty)
        return n, out

    never = fb.Context()
    try:
        want = run(never, False)
    finally:
        never.close()
    assert run(ctx, True) == want


def test_refusals_leave_the_state_unchanged(ctx):
    import oracle_binding as ob

    rng, sc, og, dyn, n_surf, quads = build(ctx, 61, n=1500, lights=2)
    # one node inside the pool's range that is not alive
    taken = set(quads) | set(n_surf) | {m for m, _ in dyn} | set(sc.lights.tolist()) | set(sc.parent.tolist())
    dead_in_range = next(n for n in range(1, sc.n) if n not in taken)
    sc.flags[dead_in_range] &= ~np.uint32(fb.NODE_ALIVE)
    ctx.set_topology(sc.parent, sc.flags, sc.mask, sc.aabb)
    ctx.update_transforms(fb.UPDATE_ALL)
    og = ob.Graph.build(sc.parent, sc.flags, sc.mask, sc.local, sc.aabb)
    og.update_hierarchical_data()
    check_frustum(ctx, og, sc, dyn, n_surf, quads)
    mesh_node = next(m for (m, k) in dyn if n_surf.get(m, 1) == 1)  # a registration, no fyx_set_node_surfaces
    multi = next(m for m, k in n_surf.items() if k > 1)  # surfaces from fyx_set_node_surfaces
    free = next(n for n in range(1, sc.n) if n not in quads and n not in n_surf and (sc.flags[n] & fb.NODE_ALIVE)
                and (n, 0) not in dyn and n not in sc.lights)
    dead = sc.n + 5
    q_node = next(iter(quads))
    good = sbo.Quad(sbo.SPRITE, SPRITE_KEYS[0], SPRITE_L)

    def refused(nodes, recs):
        with pytest.raises(fb.FyxError) as e:
            ctx.set_sprites(np.array(nodes, np.uint32), np.array([r.record() for r in recs], Context.SPRITE))
        assert e.value.code == fb._lib.FYX_ERR_INVALID_ARGUMENT

    bad_kind = good.record()
    bad_kind["kind"] = 7
    with pytest.raises(fb.FyxError) as e:
        ctx.set_sprites(np.array([free], np.uint32), np.array([bad_kind], Context.SPRITE))
    assert e.value.code == fb._lib.FYX_ERR_INVALID_ARGUMENT
    refused([dead], [good])  # out of range
    refused([dead_in_range], [good])  # in range, not alive
    refused([free, free], [good, good])  # listed twice
    refused([mesh_node], [good])  # has a registration
    refused([multi], [good])  # has surfaces
    refused([free], [sbo.Quad(sbo.SPRITE, 1 << 24, SPRITE_L)])  # key out of range
    refused([free], [sbo.Quad(sbo.SPRITE, SPRITE_KEYS[0], 1 << 16)])  # id out of range
    refused([free], [sbo.Quad(sbo.RECTANGLE, 40, SPRITE_L)])  # the sprites' layout id with another layout
    refused([free], [sbo.Quad(sbo.SPRITE, 0, SPRITE_L)])  # a registrations' key (layout 0) with another layout id
    refused([free], [sbo.Quad(sbo.SPRITE, 30, 0)])  # a registrations' layout id (another layout)
    refused([free, q_node], [sbo.Quad(sbo.SPRITE, 50, 9), sbo.Quad(sbo.RECTANGLE, 51, 9)])  # one new id, two layouts
    refused([free, q_node], [good, sbo.Quad(sbo.RECTANGLE, SPRITE_KEYS[1], RECT_L)])  # the second record fails: nothing is set
    # a quad node takes no registration
    with pytest.raises(fb.FyxError) as e:
        ctx.add_dynamic_surface(q_node, 0, SPRITE_KEYS[0], SPRITE_L, SPRITE_LAYOUT, bytes(120), np.zeros((1, 3), np.uint32))
    assert e.value.code == fb._lib.FYX_ERR_INVALID_ARGUMENT
    check_frustum(ctx, og, sc, dyn, n_surf, quads)  # nothing changed
    # a node with a skinned surface does not become a quad node
    ctx.add_skinned_surface(free, np.array([1], np.uint32), np.eye(4, dtype=f32).reshape(1, 16), None, n_verts=0)
    refused([free], [good])
    # a key and an id are free again once nothing uses them
    ctx.clear_sprites()
    ctx.clear_dynamic_surfaces()
    ctx.set_sprites(np.array([q_node], np.uint32), np.array([sbo.Quad(sbo.RECTANGLE, 0, 0).record()], Context.SPRITE))


def test_c_abi_matches_the_wrapper(ctx):
    """fyx_set_sprites and fyx_get_dynamic_batches called through ctypes directly give what the wrapper gives."""
    _, sc, og, dyn, n_surf, quads = build(ctx, 71, n=1500, lights=2)
    nodes = np.array(sorted(quads), np.uint32)
    rec = np.array([quads[n].record() for n in nodes.tolist()], Context.SPRITE)
    rec["size"] *= 2
    assert ctx._lib.fyx_set_sprites(ctx._h, len(nodes), nodes.ctypes.data_as(C.c_void_p), rec.ctypes.data_as(C.c_void_p)) == 0
    for n in nodes.tolist():
        quads[n].size = float(f32(quads[n].size) * 2)
    got, _ = check_frustum(ctx, og, sc, dyn, n_surf, quads)
    out = fb._lib.fyx_dynamic_batches()
    assert ctx._lib.fyx_get_dynamic_batches(ctx._h, 0, C.byref(out)) == 0
    assert out.n_bundles == got["bundles"].size and out.n_instances == got["instances"].size and out.n_streams == len(got["streams"])
    raw = C.string_at(out.bundles, out.n_bundles * Context.DYNAMIC_BUNDLE.itemsize)
    assert raw == got["bundles"].tobytes()
    for k in range(out.n_streams):
        st = out.streams[k]
        assert C.string_at(st.vertices, st.n_vertices * st.stride) == got["streams"][st.layout_id]["vertices"].tobytes()


def test_two_hundred_thousand_quads(ctx):
    """Over 200 000 quad nodes in one frustum: more items than one CTA of k_dyn_order covers in one chunk, many bitmap words
    per thread; then a view that gives every node one sort index, so each bundle's runs span chunks."""
    rng = np.random.default_rng(81)
    sc = ShadowScene(rng, 300_000, 4, spread=12.0, depth_z=(-30.0, -2.0), kinds=(1, 2), p_cast=0.9)
    in_view(rng, sc)
    og = sc.load(ctx)
    dyn, n_surf = register(ctx, rng, sc, n_meshes=2000)
    quads = add_quads(ctx, rng, sc, n_surf, dyn, p=0.8, sprite_meshes=500)
    ctx.update_transforms(fb.UPDATE_ALL)
    ctx.enable_instances()
    assert len(quads) >= 200_000
    got, _ = check_frustum(ctx, og, sc, dyn, n_surf, quads)
    assert got["instances"].size > 10_000
    flat = np.eye(4, dtype=f32)
    flat[2, :] = (0.0, 0.0, 0.0, -5.0)
    got, _ = check_frustum(ctx, og, sc, dyn, n_surf, quads, view=flat.T.reshape(16).copy())
    assert got["bundles"].size <= 10 and (got["bundles"]["count"] > 1024).any()


def test_scene_mirror_end_to_end(ctx):
    from fyrox_b200 import scene

    g = scene.Graph(ctx)
    a = scene.SpriteBuilder().with_size(3.0).with_color((1, 2, 3, 4)).with_material(7).build(g)
    # one batch key per (material, Forward) holds one layout: the rectangle has a material of its own
    b = scene.RectangleBuilder().with_flip_x(True).with_uv_rect((0.0, 0.0, 0.5, 0.5)).with_material(5).build(g)
    c = scene.SpriteBuilder(scene.BaseBuilder().with_cast_shadows(False)).build(g)  # drawn in no pass
    for h, z in ((a, -5.0), (b, -6.0), (c, -7.0)):
        g[h].local_transform_mut().set_position((0.5, 0.0, z))
    g.update_hierarchical_data()
    ctx.enable_instances()
    fo, ff = camera_frustum(zfar=150.0)

    def pack():
        ctx.cull([ff])
        inst = ctx.pack_instances(0, EYE, EYE)
        assert inst["node"].size == 0  # quad nodes are never instances
        return ctx.dynamic_batches("frustum", 0)

    def want(handles=None):
        """What the mirror's quad nodes push (sort indices all 0: the streams do not depend on them, and the test's nodes give
        one bundle per batch key)."""
        by_index = {h.index: g[h] for h in (handles or (a, b, c))}
        qs = {}
        for i, n in by_index.items():
            attrs = tuple(scene.SPRITE_VERTEX_ATTRIBUTES if n.kind == "sprite" else scene.RECTANGLE_VERTEX_ATTRIBUTES)
            qs[i] = sbo.Quad(scene.QUAD_KINDS[n.kind], g._batch_keys[(n.material, 1)], g._layout_ids[attrs], tuple(n.uv_rect.tolist()),
                             n.color, float(n.size), float(n.rotation), n.flip_x, n.flip_y)
        return dbo.dynamic_pass(sorted(qs), lambda i: 1, {}, lambda i: 0, lambda i: np.asarray(by_index[i].global_transform(), f32), qs,
                                False, lambda i: by_index[i].cast_shadows)[0]

    sprite_l = g._layout_ids[tuple(scene.SPRITE_VERTEX_ATTRIBUTES)]
    d = pack()
    assert d["instances"]["node"].tolist() == [a.index, b.index]
    sa = d["streams"][sprite_l]["vertices"].reshape(-1, 40)
    assert sa.shape[0] == 4 and sa[0, 20:24].view(f32)[0] == f32(3.0) and sa[0, 36:].tolist() == [1, 2, 3, 4]
    for l, st in want()["streams"].items():
        assert d["streams"][l]["vertices"].tobytes() == st["vertices"].tobytes()
    # a setter is picked up by the next sync; a removed quad node drops out
    g[a].set_color((9, 9, 9, 9))
    g[b].set_material(8)
    g.update_hierarchical_data()
    d = pack()
    assert d["streams"][sprite_l]["vertices"].reshape(-1, 40)[0, 36:].tolist() == [9] * 4
    assert d["bundles"]["batch_key"].tolist() == [g._batch_keys[(7, 1)], g._batch_keys[(8, 1)]]
    g.remove_node(a)
    g.update_hierarchical_data()
    assert pack()["instances"]["node"].tolist() == [b.index]

    # Dynamic meshes despawned and quad nodes spawned before the next sync: the pool hands the freed indices out again, and
    # the sync clears what the meshes left there (their registrations; the two-surface mesh's surface list)
    lay = [("position", 12), ("uv", 8)]

    def surf(n):
        v = np.random.default_rng(n).uniform(-1, 1, (n, 5)).astype(f32)
        return scene.Surface(vertex_buffer=v.view(np.uint8).reshape(-1), layout=lay, triangles=np.arange(n, dtype=np.uint32).reshape(-1, 3))

    meshes = []
    for k in (1, 2):
        m = scene.Node("mesh")
        m.frustum_culling = False
        m.batching_mode = scene.BatchingMode.DYNAMIC
        m.surfaces = [surf(6 + 3 * j) for j in range(k)]
        meshes.append(g.add_node(m))
    g.update_hierarchical_data()
    assert g._layout_ids[tuple(lay)] in pack()["streams"]
    freed = sorted(h.index for h in meshes)
    for h in meshes:
        g.remove_node(h)
    s1 = scene.SpriteBuilder().with_size(2.0).with_color((5, 6, 7, 8)).build(g)
    s2 = scene.RectangleBuilder().with_material(5).with_flip_y(True).build(g)
    assert sorted([s1.index, s2.index]) == freed
    g[s1].local_transform_mut().set_position((0.25, 0.5, -4.0))
    g[s2].local_transform_mut().set_position((-0.5, 0.0, -3.0))
    g.update_hierarchical_data()
    d = pack()  # no ordinary instance either (checked inside)
    w = want([b, s1, s2])
    assert sorted(d["streams"]) == sorted(w["streams"]) and g._layout_ids[tuple(lay)] not in d["streams"]
    for l, st in w["streams"].items():
        assert d["streams"][l]["vertices"].tobytes() == st["vertices"].tobytes()
        assert d["streams"][l]["triangles"].tolist() == st["triangles"].tolist()
    assert d["instances"]["node"].tolist() == w["instances"]["node"].tolist()
