"""Dynamic batching on the device: each pack's dynamic batches (bundles, instances, transformed vertex streams, shifted
triangles) against tests/dynamic_batch_oracle.py run over the same pass in DFS order, for a camera frustum (with and without
fyx_set_dfs_order) and every shadow map; registered surfaces leave the ordinary instances; register-then-clear changes nothing;
registrations follow their nodes across fyx_set_topology, and a node removed and brought back has neither its registrations
nor its surfaces; a registered surface that fyx_set_node_surfaces later removes or names skinned is pushed again; the device
getters equal the host getters."""
import numpy as np
import pytest

import dynamic_batch_oracle as dbo
import fyrox_b200 as fb
from helpers import camera_frustum, preorder_rank
from test_gpu_instance_pack import launches
from test_gpu_shadow_casters import ShadowScene, in_view
from test_gpu_shadow_instances import shadow_cull

pytestmark = pytest.mark.gpu

f32 = np.float32
NONE = dbo.NONE
EYE = np.eye(4, dtype=f32).reshape(16)
LAYOUTS = {0: (48, 0, 12, 24), 1: (15, 3, NONE, NONE)}  # the second has an odd stride: records are not 4-byte aligned


def random_surface(rng, key):
    layout_id = key % 2
    layout = LAYOUTS[layout_id]
    n = int(rng.integers(3, 40))
    raw = rng.integers(0, 256, (n, layout[0]), dtype=np.uint8)
    for off in layout[1:]:  # finite attribute values
        if off != NONE:
            w = 16 if off == layout[3] else 12
            raw[:, off:off + w] = rng.uniform(-3, 3, (n, w // 4)).astype(f32).view(np.uint8)
    tris = rng.integers(0, n, (int(rng.integers(1, 20)), 3)).astype(np.uint32)
    return dbo.DynSurface(key, layout_id, layout, raw.tobytes(), tris)


def register(ctx, rng, sc, n_meshes=300, n_keys=6, add=True, keep_one=False, exclude=()):
    """Meshes of 1-3 surfaces, about half of them batched (add=False: the same surfaces, none registered; keep_one: 2-3
    surfaces, the last never batched, so every mesh keeps an ordinary instance); returns ({(node, k): DynSurface},
    {node: n_surfaces})."""
    renderable = np.flatnonzero((sc.flags & fb.NODE_RENDERABLE) != 0)
    renderable = np.setdiff1d(renderable[renderable > 0], np.asarray(exclude, np.int64))
    meshes = rng.choice(renderable, n_meshes, replace=False).tolist()
    n_surf, dyn = {}, {}
    lists = []
    for m in meshes:
        k = int(rng.integers(2 if keep_one else 1, 4))
        n_surf[m] = k
        lists.append([(int(rng.integers(0, 5)), None) for _ in range(k)])
    ctx.set_node_surfaces(meshes, lists)
    for m in meshes:
        for k in range(n_surf[m] - (1 if keep_one else 0)):
            if rng.random() < 0.55:
                s = random_surface(rng, int(rng.integers(0, n_keys)))
                if add:
                    ctx.add_dynamic_surface(m, k, s.batch_key, s.layout_id, s.layout, s.vertices, s.triangles)
                dyn[(m, k)] = s
    return dyn, n_surf


def expect(og, order, dyn, n_surf, view, sort_of=None, quads=None, shadow=False, flags=None):
    """The oracle's pass over `order` (the pass's nodes in push order); the quad nodes' gates take the pass kind and the nodes'
    flags."""
    return dbo.dynamic_pass([int(n) for n in order], lambda n: n_surf.get(n, 1), dyn, sort_of or (lambda n: og.instance(n, view, EYE)[0]),
                            lambda n: np.asarray(og.global_transform(n), f32), quads, shadow,
                            lambda n: bool(flags[n] & fb.NODE_CAST_SHADOWS))


def push_order(nodes, rank=None):
    """The order in which the pass pushes `nodes`: DFS rank when fyx_set_dfs_order was given, else node index."""
    order = sorted(int(n) for n in nodes)
    return order if rank is None else sorted(order, key=lambda n: rank[n])


def assert_same(got, want, what):
    assert got["bundles"].tobytes() == want["bundles"].tobytes(), (what, got["bundles"][:8], want["bundles"][:8])
    assert got["instances"].tobytes() == want["instances"].tobytes(), (what, got["instances"][:8], want["instances"][:8])
    assert sorted(got["streams"]) == sorted(want["streams"]), what
    for l, st in want["streams"].items():
        g = got["streams"][l]
        assert g["stride"] == st["stride"], what
        assert g["triangles"].tolist() == st["triangles"].tolist(), (what, l)
        assert g["vertices"].tobytes() == st["vertices"].tobytes(), (what, l)


def build(ctx, seed, n=3000, lights=12):
    rng = np.random.default_rng(seed)
    sc = ShadowScene(rng, n, lights, spread=12.0, depth_z=(-30.0, -2.0), kinds=(1, 2), p_cast=1.0)
    in_view(rng, sc)
    og = sc.load(ctx)
    ctx.set_bundle_ids(rng.integers(0, 5, sc.n).astype(np.uint32))
    dyn, n_surf = register(ctx, rng, sc)
    ctx.update_transforms(fb.UPDATE_ALL)
    ctx.enable_instances()
    return rng, sc, og, dyn, n_surf


def check_frustum(ctx, og, dyn, n_surf, rank=None, view=None, cull=True):
    """The camera frustum's pass; the nodes and their order come from the oracle's own DFS (og.from_graph, pre-order): as it
    is with fyx_set_dfs_order, by node index without.  cull=False packs the last cull's list again."""
    fo, ff = camera_frustum(zfar=150.0)
    if cull:
        ctx.cull([ff])
    if view is None:
        view = np.eye(4, dtype=f32)
        view[:3, 3] = (0.5, -0.25, 2.0)
        view = view.T.reshape(16).copy()
    inst = ctx.pack_instances(0, view, np.eye(4, dtype=f32).reshape(16))
    dfs = [int(n) for n in og.from_graph(fo)]
    assert sorted(dfs) == sorted(ctx.get_visible(0).tolist())
    want, pushed = expect(og, dfs if rank is not None else sorted(dfs), dyn, n_surf, view)
    got = ctx.dynamic_batches("frustum", 0)
    assert_same(got, want, "frustum")
    assert_same(ctx.dynamic_batches("frustum", 0, device=True), want, "frustum device")
    assert sorted(zip(inst["node"].tolist(), inst["surface"].tolist())) == sorted(pushed)
    assert want["instances"].size > 20 and len(want["streams"]) == 2
    return got


@pytest.mark.parametrize("dfs", [False, True])
def test_camera_frustum_matches_the_oracle(ctx, dfs):
    _, sc, og, dyn, n_surf = build(ctx, 31 + dfs)
    rank = None
    if dfs:
        rank = preorder_rank(sc.parent)
        ctx.set_dfs_order(rank)
    check_frustum(ctx, og, dyn, n_surf, rank)


def test_every_shadow_map_matches_the_oracle(ctx):
    _, sc, og, dyn, n_surf = build(ctx, 40)
    maps, entries, want_maps = shadow_cull(ctx, og, sc)
    assert len(maps) >= 4
    total = 0
    for k, (m, w) in enumerate(zip(maps, want_maps)):
        nodes = w[4]  # the oracle's set of the map (shadow_cull checks the device's against it)
        assert np.array_equal(np.sort(entries[m["first"]: m["first"] + m["count"]]), nodes)
        want, pushed = expect(og, push_order(nodes), dyn, n_surf, w[5])
        assert_same(ctx.dynamic_batches("shadow", k), want, ("map", k))
        assert_same(ctx.dynamic_batches("shadow", k, device=True), want, ("map device", k))
        inst = ctx.get_shadow_instances(k)
        assert sorted(zip(inst["node"].tolist(), inst["surface"].tolist())) == sorted(pushed), k
        total += want["instances"].size
    assert total > 50


def canonical(inst):
    """An instance pack's outputs with each bundle's instances in a fixed order (the pack leaves that order unspecified)."""
    rows = sorted(zip(inst["node"].tolist(), inst["surface"].tolist(), inst["sort_index"].tolist(), map(bytes, inst["world"]),
                      map(bytes, inst["wvp"])))
    return rows, inst["bundles"].tobytes()


def test_register_then_clear_changes_nothing(ctx):
    """Every pack output and launch count equals that of a context that never had a dynamic surface."""
    fo, ff = camera_frustum(zfar=150.0)
    view = np.eye(4, dtype=f32).reshape(16)

    def run(c, add):
        rng = np.random.default_rng(50)
        sc = ShadowScene(rng, 3000, 12, spread=12.0, depth_z=(-30.0, -2.0), kinds=(1, 2), p_cast=1.0)
        in_view(rng, sc)
        sc.load(c)
        register(c, rng, sc, add=add)
        c.update_transforms(fb.UPDATE_ALL)
        c.enable_instances()
        c.cull([ff])
        if add:
            c.pack_instances(0, view, view)
            assert c.dynamic_batches("frustum", 0)["instances"].size > 0
            c.clear_dynamic_surfaces()
        c.cull_shadow_casters(0, np.zeros(3, f32), 200.0, 200.0, 1, 1)
        c.pack_instances(0, view, view)
        n = [launches(c, lambda: c.pack_instances(0, view, view)), launches(c, c.pack_shadow_instances)]
        n_maps = len(c.get_shadow_maps()[0])
        out = [canonical(c.pack_instances(0, view, view))] + [canonical(c.get_shadow_instances(k)) for k in range(n_maps)]
        empty = [c.dynamic_batches("frustum", 0)] + [c.dynamic_batches("shadow", k) for k in range(n_maps)]
        assert all(e["bundles"].size == 0 and not e["streams"] for e in empty)
        return n, out

    never = fb.Context()
    try:
        want = run(never, False)
    finally:
        never.close()
    assert run(ctx, True) == want


def test_registrations_and_surfaces_follow_their_nodes_across_topology(ctx):
    _, sc, og, dyn, n_surf = build(ctx, 60)
    parents = set(sc.parent.tolist())
    dyn_nodes = sorted({n for n, _ in dyn} - parents)  # leaves: removing them leaves every other node's path as it was
    gone = dyn_nodes[: len(dyn_nodes) // 3]
    flags = sc.flags.copy()
    flags[gone] &= ~np.uint32(fb.NODE_ALIVE)
    ctx.set_topology(sc.parent, flags, sc.mask, sc.aabb)
    ctx.update_transforms(fb.UPDATE_ALL)
    import oracle_binding as ob

    og2 = ob.Graph.build(sc.parent, flags, sc.mask, sc.local, sc.aabb)
    og2.update_hierarchical_data()
    kept = {k: v for k, v in dyn.items() if k[0] not in set(gone)}
    check_frustum(ctx, og2, kept, n_surf)
    # and back: the removed nodes come back (with their local matrices sent again) without registrations, and with the
    # default single surface instead of the surfaces they had
    ctx.set_topology(sc.parent, sc.flags, sc.mask, sc.aabb)
    back = np.array(gone, np.uint32)
    ctx.set_local_matrices(sc.local[back], back)
    ctx.update_transforms(fb.UPDATE_ALL)
    assert any(n_surf.get(n, 1) > 1 for n in gone)
    check_frustum(ctx, og, kept, {**n_surf, **{n: 1 for n in gone}})


def test_node_surfaces_changed_after_a_pack(ctx):
    """Surface 1 registered on two-surface meshes, one pack, then fyx_set_node_surfaces cuts some of the meshes to one surface
    and names surface 1 of the others skinned: the next pack of the same list (a skinned mesh's box is its bones', which the
    oracle's graph does not have) batches neither and pushes the skinned ones, as the oracle does."""
    rng, sc, og, dyn, n_surf = build(ctx, 100)
    meshes = [m for m, k in n_surf.items() if k == 2 and (m, 1) in dyn]
    cut, skin = meshes[0::2], meshes[1::2]
    check_frustum(ctx, og, dyn, n_surf)
    ctx.set_node_surfaces(cut, [[(int(rng.integers(0, 5)), None)] for _ in cut])
    sids = [ctx.add_skinned_surface(m, np.array([1], np.uint32), EYE.reshape(1, 16), None, n_verts=0) for m in skin]
    ctx.set_node_surfaces(skin, [[(int(rng.integers(0, 5)), None), (int(rng.integers(0, 5)), sid)] for sid in sids])
    n_surf.update({m: 1 for m in cut})
    kept = {p: s for p, s in dyn.items() if p[1] != 1 or p[0] not in set(meshes)}
    check_frustum(ctx, og, kept, n_surf, cull=False)
    vis = set(ctx.get_visible(0).tolist())
    assert len(vis & set(cut)) > 3 and len(vis & set(skin)) > 3  # the pass meets both kinds of change


def test_refusals(ctx):
    _, sc, og, dyn, n_surf = build(ctx, 70, n=500, lights=2)
    (m, k), s = next(iter(dyn.items()))

    def code(*a):
        with pytest.raises(fb.FyxError) as e:
            ctx.add_dynamic_surface(*a)
        return e.value.code

    big = dbo.DynSurface(s.batch_key, s.layout_id, s.layout, bytes(256 * s.layout[0]), np.zeros((1, 3), np.uint32))
    free = next(n for n in range(1, sc.n) if n not in n_surf and (sc.flags[n] & fb.NODE_ALIVE))
    E = fb.FyxError
    for args in [(free, 0, s.batch_key, s.layout_id, s.layout, big.vertices, big.triangles),  # 256 vertices
                 (m, k, s.batch_key, s.layout_id, s.layout, s.vertices, s.triangles),  # registered already
                 (free, 1, s.batch_key, s.layout_id, s.layout, s.vertices, s.triangles),  # no such surface
                 (free, 0, 1000, s.layout_id, (s.layout[0], NONE, NONE, NONE), s.vertices, s.triangles),  # layout id, other layout
                 (free, 0, s.batch_key, 7, (s.layout[0], NONE, NONE, NONE), s.vertices, s.triangles)]:  # key, other layout id
        assert code(*args) == fb._lib.FYX_ERR_INVALID_ARGUMENT, args[:5]
    sid = ctx.add_skinned_surface(free, np.array([1], np.uint32), np.eye(4, dtype=f32).reshape(1, 16), None, n_verts=0)
    ctx.set_node_surfaces([free], [[(0, sid)]])
    assert code(free, 0, s.batch_key, s.layout_id, s.layout, s.vertices, s.triangles) == fb._lib.FYX_ERR_INVALID_ARGUMENT
    with pytest.raises(E) as e:
        ctx.dynamic_batches("frustum", 0)
    assert e.value.code == fb._lib.FYX_ERR_STATE


def test_scale_every_chunked_path(ctx):
    """About 40 000 dynamic nodes (more than 32 bitmap words per thread of k_dyn_order) and tens of thousands of items, runs
    and bundles in one segment; then a view that gives every node one sort index, so that each bundle's runs span chunks."""
    rng = np.random.default_rng(80)
    sc = ShadowScene(rng, 150_000, 4, spread=12.0, depth_z=(-30.0, -2.0), kinds=(1, 2), p_cast=1.0)
    in_view(rng, sc)
    og = sc.load(ctx)
    dyn, n_surf = register(ctx, rng, sc, n_meshes=60_000)
    ctx.update_transforms(fb.UPDATE_ALL)
    ctx.enable_instances()
    assert len({n for n, _ in dyn}) > 33_000
    got = check_frustum(ctx, og, dyn, n_surf)
    assert got["bundles"].size > 2048 and got["instances"].size > 2048
    flat = np.eye(4, dtype=f32)
    flat[2, :] = (0.0, 0.0, 0.0, -5.0)  # view z = -5 everywhere
    got = check_frustum(ctx, og, dyn, n_surf, view=flat.T.reshape(16).copy())
    assert got["bundles"].size <= 6 and got["instances"].size > 2048
    assert (got["bundles"]["count"] > 1024).any()


def test_scene_observers_match_the_oracle(ctx):
    from test_gpu_observers import ObserverScene, observe

    rng = np.random.default_rng(90)
    s = ObserverScene(rng, 3000, 4, 2)
    og = s.load(ctx)
    dyn, n_surf = register(ctx, rng, s.sc, exclude=np.concatenate([s.cam_nodes, s.probe_nodes]))
    ctx.update_transforms(fb.UPDATE_ALL)
    ctx.enable_instances()
    table, entries, _, want_obs = observe(ctx, og, s)
    ctx.pack_scene_observer_instances()
    total = 0
    for o, (r, w) in enumerate(zip(table, want_obs)):
        want, pushed = expect(og, push_order(w["visible"]), dyn, n_surf, np.asarray(w["view"], f32).reshape(16))
        assert_same(ctx.dynamic_batches("observer", o), want, ("observer", o))
        assert_same(ctx.dynamic_batches("observer", o, device=True), want, ("observer device", o))
        inst = ctx.get_scene_observer_instances(o)
        assert sorted(zip(inst["node"].tolist(), inst["surface"].tolist())) == sorted(pushed), o
        total += want["instances"].size
    assert total > 20


def test_observers_shadow_maps_with_cascades_lod_and_static_batches(ctx):
    """The maps of fyx_cull_scene_shadow_casters: spot, point and cascaded maps, each with its own LOD filter and static-batch
    pruning.  Every batched mesh keeps one ordinary surface, whose instance gives the node's sort index for the map."""
    from test_gpu_observers import ObserverScene, observe
    from test_gpu_scene_shadows import WIDE, shadowy

    rng = np.random.default_rng(91)
    s = ObserverScene(rng, 3000, 3, 1)
    shadowy(s)
    og = s.load(ctx)
    dyn, n_surf = register(ctx, rng, s.sc, keep_one=True, exclude=np.concatenate([s.cam_nodes, s.probe_nodes]))
    ctx.update_transforms(fb.UPDATE_ALL)
    ctx.enable_instances()
    observe(ctx, og, s)
    ctx.cull_scene_shadow_casters(*WIDE, csm_enabled=True)
    ctx.pack_shadow_instances()
    maps, entries = ctx.get_shadow_maps()
    assert len(maps) >= 4 and int(maps["cascade"].max()) >= 1  # cascaded maps among them
    total = 0
    for k, m in enumerate(maps):
        inst = ctx.get_shadow_instances(k)
        sort_of = dict(zip(inst["node"].tolist(), inst["sort_index"].tolist()))
        nodes = entries[m["first"]: m["first"] + m["count"]]
        want, pushed = expect(og, push_order(nodes), dyn, n_surf, None, sort_of=lambda n: sort_of[n])
        assert_same(ctx.dynamic_batches("shadow", k), want, ("map", k))
        assert sorted(zip(inst["node"].tolist(), inst["surface"].tolist())) == sorted(pushed), k
        total += want["instances"].size
    assert total > 20


def test_getters_interleaved_across_packs(ctx):
    """Host and device getters of three packs, called in mixed order, return what a getter straight after each pack returned."""
    _, sc, og, dyn, n_surf = build(ctx, 95)
    fo0, ff0 = camera_frustum(zfar=150.0)
    fo1, ff1 = camera_frustum(target=(0.2, 0.1, -1.0), fovy=np.deg2rad(40.0), zfar=60.0)
    ctx.cull([ff0, ff1])
    ctx.cull_shadow_casters(0, np.zeros(3, f32), 200.0, 200.0, 1, 1)
    view = np.eye(4, dtype=f32).reshape(16)

    def read(kind, i, device):
        d = ctx.dynamic_batches(kind, i, device=device)
        return d["bundles"].tobytes(), d["instances"].tobytes(), [(l, st["vertices"].tobytes(), st["triangles"].tobytes())
                                                                    for l, st in sorted(d["streams"].items())]

    want = {}
    for f in (0, 1):
        ctx.pack_instances(f, view, view)
        want[("frustum", f)] = read("frustum", f, False)
    ctx.pack_shadow_instances()
    n_maps = len(ctx.get_shadow_maps()[0])
    for k in range(n_maps):
        want[("shadow", k)] = read("shadow", k, False)
    assert sum(len(want[("shadow", k)][1]) for k in range(n_maps)) > 0 and len(want[("frustum", 0)][1]) > 0
    keys = list(want) * 2
    order = np.random.default_rng(5).permutation(len(keys))
    for j in order.tolist():
        kind, i = keys[j]
        for device in ((j % 2) == 0, (j % 2) == 1):
            assert read(kind, i, device) == want[(kind, i)], (kind, i, device)


def test_scene_mirror_registers_what_the_reference_batches(ctx):
    """fyrox_b200.scene.Graph's sync registers the batched surfaces (and only those) and keeps them in step with the meshes."""
    from fyrox_b200 import scene

    g = scene.Graph(ctx)
    lay = [("position", 12), ("uv", 8)]

    def surf(n, material=0, **kw):
        v = np.random.default_rng(n).uniform(-1, 1, (n, 5)).astype(f32)
        return scene.Surface(vertex_buffer=v.view(np.uint8).reshape(-1), layout=lay, material=material,
                             triangles=np.arange(n // 3 * 3, dtype=np.uint32).reshape(-1, 3), **kw)

    def mesh(surfaces, mode, shapes=False):
        n = scene.Node("mesh")
        n.frustum_culling = False
        n.batching_mode = mode
        n.surfaces = surfaces
        if shapes:
            surfaces[0].blend_shapes_container = scene.BlendShapesContainer([scene.BlendShape()])
        return g.add_node(n)

    a = mesh([surf(6), surf(9), surf(300)], scene.BatchingMode.DYNAMIC)  # the third has 300 vertices: pushed
    b = mesh([surf(6)], scene.BatchingMode.DYNAMIC, shapes=True)  # blend shapes: pushed
    c = mesh([surf(6)], scene.BatchingMode.NONE)
    g.update_hierarchical_data()
    ctx.enable_instances()
    fo, ff = camera_frustum(zfar=150.0)

    def pack():
        ctx.cull([ff])
        inst = ctx.pack_instances(0, np.eye(4, dtype=f32).reshape(16), np.eye(4, dtype=f32).reshape(16))
        return sorted(zip(inst["node"].tolist(), inst["surface"].tolist())), ctx.dynamic_batches("frustum", 0)

    pushed, d = pack()
    assert pushed == [(a.index, 2), (b.index, 0), (c.index, 0)]
    sa = g[a].surfaces
    assert d["streams"][0]["vertices"].tobytes() == sa[0].vertex_buffer.tobytes() + sa[1].vertex_buffer.tobytes()
    assert d["instances"][["node", "triangle_offset", "triangle_count"]].tolist() == [(a.index, 0, 5)]
    g[c].batching_mode = scene.BatchingMode.DYNAMIC  # a mode change is picked up by the next sync
    g[c].surfaces[0].material = 3
    g.update_hierarchical_data()
    pushed, d = pack()
    assert pushed == [(a.index, 2), (b.index, 0)]
    assert d["bundles"]["count"].tolist() == [1, 1] and d["instances"]["node"].tolist() == [a.index, c.index]
