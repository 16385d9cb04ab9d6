"""GPU parity: the CUDA path (through the C ABI) against the oracle on the same seeded inputs.
Bit-exact for matrices, boxes, flags, palettes and skinned streams; identical visible SETS."""
import numpy as np
import pytest

import fyrox_b200 as fb
import oracle_binding as ob
from fyrox_b200.scenegen import Scene
from helpers import (NONE, preorder_rank, UNIT_BOX, assert_same_hierarchy, assert_same_visible, camera_frustum, cube_frusta, random_graph,
                     scene_pair)

pytestmark = pytest.mark.gpu


def reachable_from_root(parent, flags):
    n = len(parent)
    alive = (flags & fb.NODE_ALIVE) != 0
    reach = np.zeros(n, bool)
    reach[0] = True
    # iterate to a fixed point (parents may come after children in index order)
    changed = True
    while changed:
        ok = alive & (parent != NONE)
        new = reach.copy()
        new[ok] |= reach[parent[ok]] & alive[parent[ok]]
        changed = bool((new != reach).any())
        reach = new
    return reach


# ---- hierarchy + boxes -------------------------------------------------------------------------------
@pytest.mark.parametrize("n,units", [(2000, 0), (30000, 0), (30000, 50)])
def test_update_matches_oracle_on_generated_scenes(ctx, n, units):
    sc = Scene(n, n_units=units, verts_per_unit=40)
    og, _ = scene_pair(sc, ctx)
    og.update_hierarchical_data()
    ctx.update_transforms(fb.UPDATE_ALL)
    assert_same_hierarchy(og, ctx)


@pytest.mark.parametrize("seed,chain", [(1, 0.0), (2, 0.3), (3, 0.9)])
def test_update_matches_oracle_on_random_forests(ctx, seed, chain):
    rng = np.random.default_rng(seed)
    parent, flags, mask, local, aabb = random_graph(rng, 3000, max_depth_bias=chain)
    og = ob.Graph.build(parent, flags, mask, local, aabb)
    og.update_hierarchical_data()
    ctx.set_topology(parent, flags, mask, aabb)
    ctx.set_local_matrices(local)
    ctx.update_transforms(fb.UPDATE_ALL)
    reach = reachable_from_root(parent, flags)
    F = ctx.get_global_flags()
    assert (((F & fb.NODE_REACHABLE) != 0) == reach).all()
    assert_same_hierarchy(og, ctx, np.nonzero(reach)[0])
    # free pool records read back as identity / default box / 0
    dead = np.nonzero((flags & fb.NODE_ALIVE) == 0)[0]
    if dead.size:
        assert (ctx.get_global_matrices(dead) == np.eye(4, dtype=np.float32).reshape(16)).all()
        assert (ctx.get_global_flags(dead) == 0).all()


def test_incremental_update_equals_process_node_messages(ctx):
    """Graph::update semantics: only changed sub-trees are recomputed; result equals the oracle's
    message-driven update, including the stale skinned-mesh box when only bones move."""
    sc = Scene(20000, n_units=30, verts_per_unit=20)
    og, _ = scene_pair(sc, ctx)
    og.update_hierarchical_data()
    ctx.update_transforms(fb.UPDATE_ALL)
    rng = np.random.default_rng(5)
    for frame in range(3):
        # animate every bone + move a few random static nodes + toggle some flags
        idx, m = sc.animate(frame)
        static_nodes = np.setdiff1d(np.arange(1, sc.capacity), idx)  # a node must not get two different matrices in one batch
        extra = rng.choice(static_nodes, 25, replace=False).astype(np.uint32)
        em = sc.local_m16[extra].copy()
        em[:, 12:15] += rng.uniform(-5, 5, (25, 3)).astype(np.float32)
        all_idx = np.concatenate([idx, extra])
        all_m = np.concatenate([m, em])
        for i, mm in zip(all_idx, all_m):
            og.set_local_matrix(int(i), mm)
        tog = rng.choice(np.arange(1, sc.capacity), 10, replace=False).astype(np.uint32)
        newf = sc.flags[tog] ^ np.uint32(fb.NODE_VISIBILITY)
        for i, f in zip(tog, newf):
            og.set_visibility(int(i), bool(f & fb.NODE_VISIBILITY))
        sc.flags[tog] = newf  # scene arrays are views of generator memory: keep them in step
        og.update()
        ctx.set_local_matrices(all_m, all_idx)
        ctx.set_flags(newf, tog)
        ctx.update_transforms(fb.UPDATE_INCREMENTAL)
        assert_same_hierarchy(og, ctx)


def test_skinned_mesh_box_quirk_matches(ctx):
    """Bones visited before the mesh contribute their new position; a mesh whose own transform did
    not change keeps its cached box (scene/mesh/mod.rs:667-689)."""
    parent = np.array([NONE, 0, 0], np.uint32)
    flags = np.array([fb.NODE_DEFAULT, fb.NODE_DEFAULT, fb.NODE_DEFAULT | fb.NODE_RENDERABLE], np.uint32)
    aabb = np.stack([UNIT_BOX, UNIT_BOX, np.array([-1, -1, -1, 1, 1, 1], np.float32)])
    local = np.tile(np.eye(4, dtype=np.float32).reshape(16), (3, 1))
    local[1] = ob.translation(10, 0, 0)
    ctx.set_topology(parent, flags, None, aabb)
    ctx.set_local_matrices(local)
    ctx.add_skinned_surface(2, [1], np.eye(4, dtype=np.float32).reshape(1, 16))
    ctx.update_transforms(fb.UPDATE_INCREMENTAL)
    assert ctx.get_world_aabbs([2])[0].tolist() == [-1, -1, -1, 10, 1, 1]
    ctx.set_local_matrices(ob.translation(20, 0, 0).reshape(1, 16), [1])
    ctx.update_transforms(fb.UPDATE_INCREMENTAL)
    assert ctx.get_world_aabbs([2])[0].tolist() == [-1, -1, -1, 10, 1, 1]  # stale, like the reference
    ctx.set_local_matrices(np.eye(4, dtype=np.float32).reshape(1, 16), [2])
    ctx.update_transforms(fb.UPDATE_INCREMENTAL)
    assert ctx.get_world_aabbs([2])[0].tolist() == [-1, -1, -1, 20, 1, 1]


# ---- cull --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fused", [False, True])
def test_cull_one_frustum_matches_oracle(ctx, fused):
    sc = Scene(60000, n_units=40, verts_per_unit=20)
    og, _ = scene_pair(sc, ctx)
    og.update_hierarchical_data()
    fo, ff = camera_frustum()
    if fused:
        ctx.update_and_cull([ff], fb.UPDATE_ALL)
    else:
        ctx.update_transforms(fb.UPDATE_ALL)
        ctx.cull([ff])
    n_vis = assert_same_visible(og, ctx, [fo])
    assert 0 < n_vis < sc.n_renderable


@pytest.mark.parametrize("fused", [False, True])
def test_cull_six_cube_faces_with_masks_and_shadow_pass(ctx, fused):
    sc = Scene(60000, n_units=40, verts_per_unit=20)
    og, _ = scene_pair(sc, ctx)
    og.update_hierarchical_data()
    fos, ffs = cube_frusta()
    cam_mask = np.array([0xFFFFFFFF, 0xFFFFFFFF, 0x0000FFFF, 0xFFFFFFFF, 0x00000001, 0xFFFFFFFF], np.uint32)
    pass_flags = np.array([fb.PASS_SHADOW] * 3 + [0] * 3, np.uint32)
    if fused:
        ctx.update_and_cull(ffs, fb.UPDATE_ALL, cam_mask, pass_flags)
    else:
        ctx.update_transforms(fb.UPDATE_ALL)
        ctx.cull(ffs, cam_mask, pass_flags)
    assert_same_visible(og, ctx, fos, cam_mask, pass_flags)


def test_cull_random_forest_with_orphans_and_dead_nodes(ctx):
    rng = np.random.default_rng(11)
    parent, flags, mask, local, aabb = random_graph(rng, 5000, p_orphan=0.03)
    og = ob.Graph.build(parent, flags, mask, local, aabb)
    og.update_hierarchical_data()
    ctx.set_topology(parent, flags, mask, aabb)
    ctx.set_local_matrices(local)
    fo, ff = camera_frustum(eye=(0, 0, 60), zfar=200.0)
    ctx.update_and_cull([ff], fb.UPDATE_ALL)
    assert_same_visible(og, ctx, [fo])
    ctx.cull([ff])
    assert_same_visible(og, ctx, [fo])


def test_cull_degenerate_boxes_and_frustum_inside_box(ctx):
    """Edge cases of Frustum::is_intersects_aabb: a huge box containing the whole frustum (corner-in-box
    fallback), an inverted default box (Mesh without vertices), NaN / inf bounds, box touching a plane."""
    n = 8
    parent = np.array([NONE] + [0] * (n - 1), np.uint32)
    flags = np.full(n, fb.NODE_DEFAULT | fb.NODE_RENDERABLE, np.uint32)
    flags[0] = fb.NODE_DEFAULT
    fm = np.finfo(np.float32).max
    aabb = np.array([
        [-0.5, -0.5, -0.5, 0.5, 0.5, 0.5],
        [-1e6, -1e6, -1e6, 1e6, 1e6, 1e6],       # contains the frustum
        [fm, fm, fm, -fm, -fm, -fm],             # AxisAlignedBoundingBox::default()
        [np.nan, 0, 0, 1, 1, 1],
        [-np.inf, -np.inf, -np.inf, np.inf, np.inf, np.inf],
        [-1, -1, -20, 1, 1, -10],                # in front of the camera
        [200, 200, 200, 201, 201, 201],          # far outside
        [-1, -1, -0.1, 1, 1, 0.0],               # touching the near plane region
    ], np.float32)
    local = np.tile(np.eye(4, dtype=np.float32).reshape(16), (n, 1))
    og = ob.Graph.build(parent, flags, None, local, aabb)
    og.update_hierarchical_data()
    ctx.set_topology(parent, flags, None, aabb)
    ctx.set_local_matrices(local)
    fo, ff = camera_frustum()
    ctx.update_and_cull([ff], fb.UPDATE_ALL)
    assert_same_hierarchy(og, ctx)
    assert_same_visible(og, ctx, [fo])
    # K4 on the GPU: identity view-projection, unit box in, [5,15]^3 out
    fo_i = ob.frustum_from_vp(np.eye(4, dtype=np.float32).reshape(16))
    ff_i = fb.frustum_from_view_projection_matrix(np.eye(4, dtype=np.float32).reshape(16))
    aabb2 = aabb.copy()
    aabb2[1] = [5, 5, 5, 15, 15, 15]
    og2 = ob.Graph.build(parent, flags, None, local, aabb2)
    og2.update_hierarchical_data()
    ctx.set_local_aabbs(aabb2)
    ctx.update_and_cull([ff_i], fb.UPDATE_ALL)
    assert_same_visible(og2, ctx, [fo_i])
    vis = set(ctx.get_visible(0).tolist())
    assert 0 not in vis and 1 not in vis and 5 not in vis and 7 in vis  # node 0 is a pivot; 7's box straddles z in [-1,1]


def test_empty_and_tiny_graphs(ctx):
    fo, ff = camera_frustum()
    ctx.set_topology(np.array([NONE], np.uint32), np.array([fb.NODE_DEFAULT], np.uint32))
    ctx.update_and_cull([ff], fb.UPDATE_ALL)
    assert ctx.get_visible(0).size == 0
    assert ctx.get_global_matrices()[0].tolist() == np.eye(4, dtype=np.float32).reshape(16).tolist()
    ctx.set_topology(np.empty(0, np.uint32), np.empty(0, np.uint32))
    ctx.update_and_cull([ff], fb.UPDATE_ALL)
    assert ctx.get_visible(0).size == 0
    ctx.cull([])


# ---- the reference's own hierarchy test, through the host mirror -----------------------------------
def test_k6_hierarchy_changes_propagation_reads_like_the_reference():
    """fyrox-impl/src/scene/graph/mod.rs:2646-2739 transcribed onto fyrox_b200.scene."""
    from fyrox_b200.scene import BaseBuilder, Graph, PivotBuilder, TransformBuilder

    graph = Graph()
    c = PivotBuilder(BaseBuilder().with_local_transform(TransformBuilder().with_local_position((0.0, 0.0, 1.0)).build())).build(graph)
    b = PivotBuilder(
        BaseBuilder().with_visibility(False).with_enabled(False)
        .with_local_transform(TransformBuilder().with_local_position((0.0, 1.0, 0.0)).build()).with_child(c)
    ).build(graph)
    d = PivotBuilder(BaseBuilder().with_local_transform(TransformBuilder().with_local_position((1.0, 1.0, 1.0)).build())).build(graph)
    a = PivotBuilder(
        BaseBuilder().with_local_transform(TransformBuilder().with_local_position((1.0, 0.0, 0.0)).build()).with_child(b).with_child(d)
    ).build(graph)
    assert (graph.root.index, graph.root.generation) == (0, 1) and (c.index, c.generation) == (1, 1)  # K10

    graph.update((1.0, 1.0), 1.0 / 60.0)
    assert graph[a].global_position().tolist() == [1.0, 0.0, 0.0]
    assert graph[b].global_position().tolist() == [1.0, 1.0, 0.0]
    assert graph[c].global_position().tolist() == [1.0, 1.0, 1.0]
    assert graph[d].global_position().tolist() == [2.0, 1.0, 1.0]
    assert graph[a].global_visibility() and not graph[b].global_visibility()
    assert not graph[c].global_visibility() and graph[d].global_visibility()
    assert graph[a].is_globally_enabled() and not graph[b].is_globally_enabled()
    assert not graph[c].is_globally_enabled() and graph[d].is_globally_enabled()

    graph[b].local_transform_mut().set_position((0.0, 2.0, 0.0))
    graph[a].set_enabled(False)
    graph[b].set_visibility(True)
    graph.update((1.0, 1.0), 1.0 / 60.0)
    assert graph[a].global_position().tolist() == [1.0, 0.0, 0.0]
    assert graph[b].global_position().tolist() == [1.0, 2.0, 0.0]
    assert graph[c].global_position().tolist() == [1.0, 2.0, 1.0]
    assert graph[d].global_position().tolist() == [2.0, 1.0, 1.0]
    assert all(graph[h].global_visibility() for h in (a, b, c, d))
    assert not any(graph[h].is_globally_enabled() for h in (a, b, c, d))
    graph.ctx.close()


def test_k7_global_scale_and_from_graph_through_the_host_mirror():
    from fyrox_b200.scene import BaseBuilder, Graph, MeshBuilder, ObserverPosition, PivotBuilder, RenderDataBundleStorage, TransformBuilder

    graph = Graph()
    c = PivotBuilder(BaseBuilder().with_local_transform(TransformBuilder().with_local_scale((1.0, 2.0, 3.0)).build())).build(graph)
    b = PivotBuilder(BaseBuilder().with_local_transform(TransformBuilder().with_local_scale((3.0, 2.0, 1.0)).build()).with_child(c)).build(graph)
    a = PivotBuilder(BaseBuilder().with_local_transform(TransformBuilder().with_local_scale((1.0, 1.0, 2.0)).build()).with_child(b)).build(graph)
    assert graph.global_scale(a).tolist() == [1.0, 1.0, 2.0]
    assert graph.global_scale(b).tolist() == [3.0, 2.0, 2.0]
    assert graph.global_scale(c).tolist() == [3.0, 4.0, 6.0]
    near = MeshBuilder(BaseBuilder().with_local_bounding_box([-1, -1, -1, 1, 1, 1])
                       .with_local_transform(TransformBuilder().with_local_position((0.0, 0.0, -10.0)).build())).build(graph)
    behind = MeshBuilder(BaseBuilder().with_local_bounding_box([-1, -1, -1, 1, 1, 1])
                         .with_local_transform(TransformBuilder().with_local_position((0.0, 0.0, 50.0)).build())).build(graph)
    noshadow = MeshBuilder(BaseBuilder().with_cast_shadows(False).with_local_bounding_box([-1, -1, -1, 1, 1, 1])
                           .with_local_transform(TransformBuilder().with_local_position((2.0, 0.0, -10.0)).build())).build(graph)
    graph.update()
    op = ObserverPosition(np.zeros(3, np.float32), 0.1, 150.0, ob.look_at_rh((0, 0, 0), (0, 0, -1), (0, 1, 0)), ob.perspective(16 / 9, np.deg2rad(60.0), 0.1, 150.0))
    main = RenderDataBundleStorage.from_graph(graph, 0xFFFFFFFF, 0.0, op, "GBuffer")
    assert set(h.index for h in main.visible_handles) == {near.index, noshadow.index}
    shadow = RenderDataBundleStorage.from_graph(graph, 0xFFFFFFFF, 0.0, op, "SpotShadow")
    assert set(h.index for h in shadow.visible_handles) == {near.index}
    assert behind.index not in set(h.index for h in main.visible_handles)
    graph.ctx.close()


def test_static_batching_through_the_host_mirror_reads_like_the_reference():
    """Mesh::set_batching_mode(BatchingMode::Static): once the mesh is rendered, collect_render_data returns
    RdcControlFlow::Break and the DFS of from_graph skips its children (scene/mesh/mod.rs:701-725, bundle.rs:996-1001);
    a static mesh outside the frustum lets the DFS go on."""
    from fyrox_b200.scene import BaseBuilder, BatchingMode, Graph, MeshBuilder, ObserverPosition, RenderDataBundleStorage, TransformBuilder

    graph = Graph()
    box = [-1, -1, -1, 1, 1, 1]
    at = lambda x, y, z: TransformBuilder().with_local_position((x, y, z)).build()
    child_a = MeshBuilder(BaseBuilder().with_local_bounding_box(box).with_local_transform(at(1.0, 0.0, 0.0))).build(graph)
    parent_a = MeshBuilder(BaseBuilder().with_local_bounding_box(box).with_local_transform(at(0.0, 0.0, -10.0)).with_child(child_a)).build(graph)
    # the same pair again, but the parent sits behind the camera while its child (local offset) is in front of it
    child_b = MeshBuilder(BaseBuilder().with_local_bounding_box(box).with_local_transform(at(0.0, 0.0, -70.0))).build(graph)
    parent_b = MeshBuilder(BaseBuilder().with_local_bounding_box(box).with_local_transform(at(0.0, 0.0, 50.0)).with_child(child_b)).build(graph)
    graph.update()
    op = ObserverPosition(np.zeros(3, np.float32), 0.1, 150.0, ob.look_at_rh((0, 0, 0), (0, 0, -1), (0, 1, 0)), ob.perspective(16 / 9, np.deg2rad(60.0), 0.1, 150.0))
    vis = lambda: set(h.index for h in RenderDataBundleStorage.from_graph(graph, 0xFFFFFFFF, 0.0, op, "GBuffer").visible_handles)
    assert vis() == {parent_a.index, child_a.index, child_b.index}
    graph[parent_a].set_batching_mode(BatchingMode.STATIC)
    graph[parent_b].set_batching_mode(BatchingMode.STATIC)
    graph.update()
    assert vis() == {parent_a.index, child_b.index}  # a rendered static batch hides its child; a culled one does not
    graph[parent_a].set_batching_mode(BatchingMode.NONE)
    graph.update()
    assert vis() == {parent_a.index, child_a.index, child_b.index}
    graph.ctx.close()


# ---- palette + skinning -------------------------------------------------------------------------------
def test_palette_and_skinning_match_oracle(ctx):
    sc = Scene(6000, n_units=24, verts_per_unit=1237)  # 1237: not a multiple of 4 ⇒ padded quads
    og, sids = scene_pair(sc, ctx)
    idx, m = sc.animate(3)
    for i, mm in zip(idx, m):
        og.set_local_matrix(int(i), mm)
    og.update_hierarchical_data()
    ctx.set_local_matrices(m, idx)
    ctx.update_transforms(fb.UPDATE_ALL)
    ctx.build_palettes()
    ctx.skin()
    max_err = 0.0
    for u, sid in enumerate(sids):
        mesh = sc.unit_mesh_node(u)
        pal_o = og.bone_matrices(mesh, 0, sc.bones_per_unit)
        pal_g = ctx.get_palette(sid)
        assert pal_g.tobytes() == pal_o.tobytes(), f"palette of unit {u} differs"
        pos_o, nrm_o = og.skin(mesh, 0, sc.verts_per_unit)
        pos_g, nrm_g = ctx.get_skinned(sid)
        max_err = max(max_err, float(np.abs(pos_g - pos_o).max()))
        assert np.abs(pos_g - pos_o).max() <= 1e-5  # the tolerance BASELINE.json's north_star states
        assert pos_g.tobytes() == pos_o.tobytes(), f"skinned positions of unit {u} are not bit-identical"
        assert nrm_g.tobytes() == nrm_o.tobytes(), f"skinned normals of unit {u} are not bit-identical"
    assert max_err == 0.0


def test_skinning_edge_cases(ctx):
    """Zero weights, repeated indices, a dead / NONE bone (identity matrix), 255 bones, 1 vertex."""
    nb = 255
    n = nb + 2
    parent = np.array([NONE] + [0] * (n - 1), np.uint32)
    flags = np.full(n, fb.NODE_DEFAULT, np.uint32)
    flags[n - 1] |= fb.NODE_RENDERABLE
    flags[7] = 0  # a dead bone node ⇒ identity palette entry
    rng = np.random.default_rng(3)
    local = np.tile(np.eye(4, dtype=np.float32).reshape(16), (n, 1))
    local[1:, 12:15] = rng.uniform(-5, 5, (n - 1, 3)).astype(np.float32)
    bones = np.arange(1, nb + 1, dtype=np.uint32)
    bones[9] = NONE
    ib = np.tile(np.eye(4, dtype=np.float32).reshape(16), (nb, 1))
    ib[:, 12:15] = rng.uniform(-1, 1, (nb, 3)).astype(np.float32)
    nv = 1001
    rec = np.zeros((nv, 68), np.uint8)
    f = rec[:, :64].view(np.float32)
    f[:, 0:3] = rng.uniform(-3, 3, (nv, 3))
    f[:, 5:8] = rng.normal(size=(nv, 3))
    w = rng.random((nv, 4)).astype(np.float32)
    w[::3, 2:] = 0.0
    w[1::7, 1:] = 0.0
    f[:, 12:16] = w / w.sum(axis=1, keepdims=True)
    bi = rng.integers(0, nb, (nv, 4)).astype(np.uint8)
    bi[::5] = bi[::5, :1]  # all four influences on the same bone
    bi[0] = [7 - 1, 9, 254, 0]  # dead bone, NONE bone, last bone, first bone
    rec[:, 64:68] = bi
    og = ob.Graph.build(parent, flags, None, local, None)
    for k in range(nb):
        if bones[k] != NONE and flags[bones[k]] & fb.NODE_ALIVE:
            og.set_inv_bind(int(bones[k]), ib[k])
    og.add_surface(n - 1, bones, rec.reshape(-1))
    og.L.orc_graph_drop_messages(og.h)
    og.update_hierarchical_data()
    ctx.set_topology(parent, flags)
    ctx.set_local_matrices(local)
    sid = ctx.add_skinned_surface(n - 1, bones, ib, rec.reshape(-1))
    sid1 = ctx.add_skinned_surface(n - 1, bones[:3], ib[:3], np.ascontiguousarray(np.concatenate([rec[:1, :64], np.zeros((1, 4), np.uint8)], axis=1)).reshape(-1))
    ctx.update_transforms(fb.UPDATE_ALL)
    ctx.build_palettes()
    ctx.skin()
    pal_o = og.bone_matrices(n - 1, 0, nb)
    pal_g = ctx.get_palette(sid)
    assert pal_g[6].tolist() == np.eye(4, dtype=np.float32).reshape(16).tolist()  # dead bone
    assert pal_g[9].tolist() == np.eye(4, dtype=np.float32).reshape(16).tolist()  # NONE bone
    assert pal_g.tobytes() == pal_o.tobytes()
    pos_o, nrm_o = og.skin(n - 1, 0, nv)
    pos_g, nrm_g = ctx.get_skinned(sid)
    assert pos_g.tobytes() == pos_o.tobytes() and nrm_g.tobytes() == nrm_o.tobytes()
    p1, _ = ctx.get_skinned(sid1)
    assert p1.shape == (1, 3)


def test_blend_shapes_ahead_of_skinning_match_oracle(ctx):
    """N4: blend-shape offsets are added to positions / normals before the skinning (standard.shader:167-173), in shape
    order, with BlendShape::weight / 100 — surfaces with and without shapes in one launch, vertex counts that are not
    multiples of the 128-vertex blocks, weight updates, removal.  Bit for bit against orc_skin_vertices_blend."""
    import ctypes as C

    sc = Scene(6000, n_units=9, verts_per_unit=1237)
    og, sids = scene_pair(sc, ctx)
    idx, m = sc.animate(2)
    for i, mm in zip(idx, m):
        og.set_local_matrix(int(i), mm)
    og.update_hierarchical_data()
    ctx.set_local_matrices(m, idx)
    rng = np.random.default_rng(12)
    nv = sc.verts_per_unit
    shapes = {}
    for u in (0, 3, 4, 8):  # the others have no blend shapes
        ns = [1, 3, 7, 2][len(shapes)]
        stride = nv + [0, 11, 300, 1][len(shapes)]  # width * height of the texture >= vertex count
        off = (rng.normal(size=(ns, stride, 9)) * 0.2).astype(np.float16)
        off[rng.random((ns, stride, 9)) < 0.6] = 0  # sparse, like the importers' index -> offset maps
        off[0, 0, :3] = [np.float16(6.1e-5), np.float16(-0.0), np.float16(5.96e-8)]  # smallest normal, -0, a subnormal
        w = rng.uniform(0, 100, ns).astype(np.float32)
        w[-1] = 0.0 if ns > 1 else 100.0
        shapes[u] = (off.view(np.uint16), w)
        ctx.set_blend_shapes(sids[u], off.view(np.uint16), w)

    def check():
        ctx.update_transforms(fb.UPDATE_ALL)
        ctx.build_palettes()
        ctx.skin()
        L = ob.lib()
        lay = ob.ANIMATED_VERTEX
        for u, sid in enumerate(sids):
            mesh = sc.unit_mesh_node(u)
            pal_o = og.bone_matrices(mesh, 0, sc.bones_per_unit)
            pos_g, nrm_g = ctx.get_skinned(sid)
            if u in shapes:
                rec, w = shapes[u]
                verts = sc.unit_vertices(u)[0]
                pos_o = np.empty((nv, 3), np.float32)
                nrm_o = np.empty((nv, 3), np.float32)
                w100 = (w / np.float32(100.0)).astype(np.float32)
                L.orc_skin_vertices_blend(ob.fp(np.ascontiguousarray(pal_o.reshape(-1))), nv, verts.ctypes.data_as(C.c_void_p), C.byref(lay), rec.shape[0],
                                          rec.ctypes.data_as(C.c_void_p), rec.shape[1], ob.fp(w100), ob.fp(pos_o.reshape(-1)), ob.fp(nrm_o.reshape(-1)))
            else:
                pos_o, nrm_o = og.skin(mesh, 0, nv)
            assert pos_g.tobytes() == pos_o.tobytes(), f"unit {u}: positions differ"
            assert nrm_g.tobytes() == nrm_o.tobytes(), f"unit {u}: normals differ"

    check()
    base0 = og.skin(sc.unit_mesh_node(0), 0, nv)[0]
    assert ctx.get_skinned(sids[0])[0].tobytes() != base0.tobytes()  # the shapes really moved something
    # new weights (Mesh::blend_shapes_mut), then fewer shapes, then none
    rec, w = shapes[4]
    w2 = rng.uniform(0, 100, len(w)).astype(np.float32)
    ctx.set_blend_shape_weights(sids[4], w2)
    shapes[4] = (rec, w2)
    check()
    rec3, w3 = shapes[3]
    shapes[3] = (np.ascontiguousarray(rec3[:2]), w3[:2].copy())
    ctx.set_blend_shapes(sids[3], shapes[3][0], shapes[3][1])
    ctx.set_blend_shapes(sids[0], np.empty((0, 0, 9), np.uint16))
    del shapes[0]
    check()
    with pytest.raises(fb.FyxError):
        ctx.set_blend_shape_weights(sids[4], w2[:1])  # wrong count
    with pytest.raises(fb.FyxError):
        ctx.set_blend_shapes(sids[1], np.zeros((1, nv - 1, 9), np.uint16))  # fewer records than vertices


def test_errors_are_reported_not_fatal(ctx):
    parent = np.array([NONE, 0], np.uint32)
    ctx.set_topology(parent, np.full(2, fb.NODE_DEFAULT, np.uint32))
    bad = np.eye(4, dtype=np.float32).reshape(16).copy()
    bad[3] = 0.5  # projective row
    ctx.set_local_matrices(bad.reshape(1, 16), [1])
    with pytest.raises(fb.FyxError) as e:
        ctx.update_transforms(fb.UPDATE_ALL)
    assert e.value.code == fb._lib.FYX_ERR_NOT_AFFINE
    ctx.update_transforms(fb.UPDATE_ALL)  # the bad matrix was skipped; the context is still usable
    assert ctx.get_global_matrices([1])[0].tolist() == np.eye(4, dtype=np.float32).reshape(16).tolist()
    with pytest.raises(fb.FyxError) as e:
        ctx.set_topology(np.array([1, 0], np.uint32), np.full(2, fb.NODE_DEFAULT, np.uint32))  # 2-cycle
    assert e.value.code == fb._lib.FYX_ERR_TOPOLOGY
    rec = np.zeros((4, 68), np.uint8)
    rec[:, 64] = 9  # bone index out of range for a 2-bone surface
    ctx.add_skinned_surface(1, [0, 1], np.tile(np.eye(4, dtype=np.float32).reshape(16), (2, 1)), rec.reshape(-1))
    with pytest.raises(fb.FyxError) as e:
        ctx.commit_surfaces()
    assert e.value.code == fb._lib.FYX_ERR_INVALID_ARGUMENT
    with pytest.raises(fb.FyxError):
        ctx.get_visible(5)


def test_render_prep_one_call_frame(ctx):
    sc = Scene(30000, n_units=30, verts_per_unit=200)
    og, sids = scene_pair(sc, ctx)
    fos, ffs = cube_frusta()
    for frame in range(2):
        idx, m = sc.animate(frame)
        for i, mm in zip(idx, m):
            og.set_local_matrix(int(i), mm)
        og.update_hierarchical_data()
        ctx.render_prep(update_flags=fb.UPDATE_ALL, changed_m16=m, changed_idx=idx, frusta=ffs)
        assert_same_hierarchy(og, ctx)
        assert_same_visible(og, ctx, fos)
        for u in (0, len(sids) - 1):
            mesh = sc.unit_mesh_node(u)
            pos_o, nrm_o = og.skin(mesh, 0, sc.verts_per_unit)
            pos_g, nrm_g = ctx.get_skinned(sids[u])
            assert pos_g.tobytes() == pos_o.tobytes() and nrm_g.tobytes() == nrm_o.tobytes()
    t = ctx.timings()
    assert t["total_ms"] > 0 and ctx.kernel_launch_count() > 0
    # pinned inputs take the zero-staging path
    pin_m = fb.PinnedBuffer((idx.size, 16), np.float32)
    pin_i = fb.PinnedBuffer((idx.size,), np.uint32)
    pin_m.array[:] = m
    pin_i.array[:] = idx
    ctx.render_prep(update_flags=fb.UPDATE_ALL, changed_m16=pin_m.ptr, changed_idx=pin_i.ptr, n_changed=idx.size, frusta=ffs)
    assert_same_visible(og, ctx, fos)
    pin_m.free()
    pin_i.free()


def test_pipelined_frames_match_oracle(ctx):
    """FYX_FRAME_ASYNC + fyx_frame_wait: two frames in flight, uploads on the copy stream; every collected
    frame equals the oracle's frame."""
    sc = Scene(30000, n_units=30, verts_per_unit=64)
    og, sids = scene_pair(sc, ctx)
    fos, ffs = cube_frusta()
    n_frames = 5
    pins = []
    for fr in range(n_frames):
        idx, m = sc.animate(fr)
        pm = fb.PinnedBuffer(m.shape, np.float32)
        pi = fb.PinnedBuffer(idx.shape, np.uint32)
        pm.array[:] = m
        pi.array[:] = idx
        pins.append((pi, pm, idx, m))

    def oracle_frame(fr):
        _, _, idx, m = pins[fr]
        for i, mm in zip(idx, m):
            og.set_local_matrix(int(i), mm)
        og.update_hierarchical_data()
        return [np.sort(og.from_graph(fo)) for fo in fos]

    def submit(fr):
        pi, pm, idx, _ = pins[fr]
        ctx.render_prep(update_flags=fb.UPDATE_ALL, changed_m16=pm.ptr, changed_idx=pi.ptr, n_changed=idx.size, frusta=ffs,
                        readback_visible=True, async_=True)

    def check(fr):
        want = oracle_frame(fr)
        for f in range(len(ffs)):
            assert np.array_equal(np.sort(ctx.get_visible(f)), want[f]), f"frame {fr} frustum {f}"

    submit(0)
    with pytest.raises(fb.FyxError):
        ctx.get_visible(0)  # still in flight
    for fr in range(1, n_frames):
        submit(fr)
        ctx.frame_wait()
        check(fr - 1)
    with pytest.raises(fb.FyxError):
        submit(0)
        submit(1)
        submit(2)  # a third frame in flight is refused
    ctx.frame_wait()
    ctx.frame_wait()
    ctx.frame_wait()  # no-op
    ctx.sync()
    for p in pins:
        p[0].free()
        p[1].free()


def _oracle_transform(pos, rot, scale, statics=None):
    tr = ob.Transform()
    ob.lib().orc_transform_identity(tr)
    tr.local_position[:] = pos.tolist()
    tr.local_rotation[:] = rot.tolist()
    tr.local_scale[:] = scale.tolist()
    if statics is not None:
        tr.pre_rotation[:] = statics[0:4].tolist()
        tr.post_rotation_matrix[:] = statics[4:13].tolist()
        tr.rotation_offset[:] = statics[13:16].tolist()
        tr.rotation_pivot[:] = statics[16:19].tolist()
        tr.scaling_offset[:] = statics[19:22].tolist()
        tr.scaling_pivot[:] = statics[22:25].tolist()
    m = np.empty(16, np.float32)
    ob.lib().orc_transform_calculate_local(tr, ob.fp(m))
    return m


@pytest.mark.parametrize("with_statics", [False, True])
def test_trs_upload_equals_calculate_local_transform(ctx, with_statics):
    """N1: Transform::calculate_local_transform on the device (fyx_set_local_trs) is bit-identical to the
    oracle's restatement of scene/transform.rs:421-540, with default and with arbitrary pivots / offsets /
    pre- and post-rotation; the hierarchy built on top matches too."""
    rng = np.random.default_rng(21 + with_statics)
    n = 4000
    parent = np.full(n, NONE, np.uint32)
    parent[1:] = (rng.random(n - 1) * np.arange(1, n)).astype(np.uint32)  # parent index < own index
    flags = np.full(n, fb.NODE_DEFAULT | fb.NODE_RENDERABLE, np.uint32)
    flags[0] = fb.NODE_DEFAULT
    pos = rng.uniform(-30, 30, (n, 3)).astype(np.float32)
    rot = rng.normal(size=(n, 4)).astype(np.float32)
    rot /= np.linalg.norm(rot, axis=1, keepdims=True)
    scale = rng.uniform(0.3, 2.0, (n, 3)).astype(np.float32)
    pos[0] = 0
    rot[0] = (0, 0, 0, 1)
    scale[0] = 1
    # exercise exact zeros / negative zeros / denormals in the inputs
    pos[5] = (0.0, -0.0, 1e-42)
    rot[6] = (0.0, 0.0, 0.0, 1.0)
    rot[7] = (1.0, 0.0, -0.0, 0.0)
    scale[8] = (1.0, -1.0, 0.0)
    statics = None
    if with_statics:
        statics = np.zeros((n, 25), np.float32)
        q = rng.normal(size=(n, 4)).astype(np.float32)
        statics[:, 0:4] = q / np.linalg.norm(q, axis=1, keepdims=True)
        post = rng.normal(size=(n, 3, 3)).astype(np.float32)
        statics[:, 4:13] = post.reshape(n, 9)
        statics[:, 13:25] = rng.uniform(-2, 2, (n, 12)).astype(np.float32)
        statics[0, :] = 0
        statics[0, 3] = 1
        statics[0, [4, 8, 12]] = 1
    local = np.stack([_oracle_transform(pos[i], rot[i], scale[i], None if statics is None else statics[i]) for i in range(n)])
    og = ob.Graph.build(parent, flags, None, local, None)
    og.update_hierarchical_data()
    ctx.set_topology(parent, flags)
    if statics is not None:
        ctx.set_transform_statics(statics)
    trs = np.concatenate([pos, rot, scale], axis=1)
    half = n // 2
    ctx.set_local_trs(trs[:half])                                    # idx NULL = nodes 0..count-1
    ctx.set_local_trs(trs[half:], np.arange(half, n, dtype=np.uint32))
    ctx.update_transforms(fb.UPDATE_ALL)
    from helpers import bits_equal

    G = ctx.get_global_matrices()
    Go = og.global_transforms()
    assert bits_equal(G, Go).all(), np.nonzero((~bits_equal(G, Go)).any(axis=1))[0][:10]
    # node 0 has no parent: its global matrix is I * local, i.e. the local matrix up to the sign of zeros
    assert np.array_equal(G[0], local[0])
    # one-call frame with TRS payload (pinned, pipelined)
    pt = fb.PinnedBuffer(trs.shape, np.float32)
    pt.array[:] = trs
    pt.array[:, 0] += 1.0
    local2 = np.stack([_oracle_transform(pt.array[i, 0:3], pt.array[i, 3:7], pt.array[i, 7:10], None if statics is None else statics[i]) for i in range(n)])
    for i in range(n):
        og.set_local_matrix(i, local2[i])
    og.update_hierarchical_data()
    ctx.render_prep(update_flags=fb.UPDATE_INCREMENTAL, changed_trs=pt.ptr, n_changed=n, frusta=[], readback_visible=False, async_=True)
    ctx.sync()
    assert bits_equal(ctx.get_global_matrices(), og.global_transforms()).all()
    # rotation-only updates (Transform::set_rotation): position / scale stay what the last full record said
    rot2 = rng.normal(size=(n, 4)).astype(np.float32)
    rot2 /= np.linalg.norm(rot2, axis=1, keepdims=True)
    some = np.sort(rng.choice(np.arange(1, n), n // 3, replace=False)).astype(np.uint32)
    for i in some:
        og.set_local_matrix(int(i), _oracle_transform(pt.array[i, 0:3], rot2[i], pt.array[i, 7:10], None if statics is None else statics[i]))
    og.update()
    ctx.set_local_rotations(rot2[some], some)
    ctx.update_transforms(fb.UPDATE_INCREMENTAL)
    assert bits_equal(ctx.get_global_matrices(), og.global_transforms()).all()
    pq = fb.PinnedBuffer((n, 4), np.float32)
    pq.array[:] = rot
    for i in range(n):
        og.set_local_matrix(i, _oracle_transform(pt.array[i, 0:3], rot[i], pt.array[i, 7:10], None if statics is None else statics[i]))
    og.update_hierarchical_data()
    ctx.render_prep(update_flags=fb.UPDATE_INCREMENTAL, changed_rot=pq.ptr, n_changed=n, frusta=[], readback_visible=False, async_=True)
    ctx.sync()
    assert bits_equal(ctx.get_global_matrices(), og.global_transforms()).all()
    pq.free()
    pt.free()


def test_cpp_host_mirror_runs_the_reference_hierarchy_tests():
    """tests/cpp/test_host.cpp: K6 / K7 / K10 and a from_graph cull through the C++ host mirror
    (fyrox_b200/host/fyrox_host.hpp), which drives the device through fyx_set_local_trs."""
    import os
    import subprocess

    d = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpp")
    r = subprocess.run(["make", "-C", d, "test_host"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    r = subprocess.run([os.path.join(d, "test_host")], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and r.stdout.strip() == "OK", r.stdout + r.stderr


def test_topology_change_keeps_surfaces_and_flag_changes_resize_nothing(ctx):
    """A second fyx_set_topology (nodes added / re-parented) with skinned surfaces already uploaded, and
    fyx_set_flags turning pivots into renderable nodes, still match an oracle rebuilt from scratch."""
    sc = Scene(8000, n_units=10, verts_per_unit=50)
    og, sids = scene_pair(sc, ctx)
    fo, ff = camera_frustum(zfar=500.0, fovy=np.deg2rad(100.0))
    ctx.update_and_cull([ff], fb.UPDATE_ALL)
    # grow the graph: 500 new meshes hanging under existing nodes, and move 100 old leaves under new parents
    rng = np.random.default_rng(9)
    n0, extra = sc.capacity, 500
    parent = np.concatenate([sc.parent, rng.integers(0, n0, extra).astype(np.uint32)])
    flags = np.concatenate([sc.flags, np.full(extra, fb.NODE_DEFAULT | fb.NODE_RENDERABLE, np.uint32)])
    mask = np.concatenate([sc.render_mask, np.full(extra, 0xFFFFFFFF, np.uint32)])
    local = np.concatenate([sc.local_m16, np.tile(ob.translation(1, 2, 3), (extra, 1))])
    aabb = np.concatenate([sc.local_aabb, np.tile(np.array([-1, -1, -1, 1, 1, 1], np.float32), (extra, 1))])
    for u in range(sc.n_units):  # keep the skinned meshes' vertex-derived boxes
        aabb[sc.unit_mesh_node(u)] = sc.unit_vertices(u)[1]
    movers = np.nonzero((sc.flags & fb.NODE_RENDERABLE) != 0)[0][:100]
    parent[movers] = np.arange(n0, n0 + 100, dtype=np.uint32)  # old leaves under the new nodes (larger indices)
    # every pivot becomes renderable through fyx_set_flags afterwards
    piv = np.nonzero((flags & fb.NODE_RENDERABLE) == 0)[0].astype(np.uint32)
    piv = piv[piv != 0]
    flags2 = flags.copy()
    flags2[piv] |= fb.NODE_RENDERABLE
    og2 = ob.Graph.build(parent, flags2, mask, local, aabb)
    for u in range(sc.n_units):
        bones = sc.unit_bone_nodes(u)
        for k, b in enumerate(bones):
            og2.set_inv_bind(int(b), sc.unit_inv_bind(u)[k])
        og2.add_surface(sc.unit_mesh_node(u), bones, sc.unit_vertices(u)[0])
    og2.L.orc_graph_drop_messages(og2.h)
    og2.update_hierarchical_data()
    ctx.set_topology(parent, flags, mask, aabb)
    ctx.set_local_matrices(local)
    ctx.set_flags(flags2[piv], piv)
    ctx.update_and_cull([ff], fb.UPDATE_INCREMENTAL)  # everything is marked changed by the new topology
    # pivots of the oracle are Base nodes (unit box); the GPU got the same unit boxes from scenegen
    reach = np.ones(len(parent), bool)
    assert_same_hierarchy(og2, ctx, np.arange(len(parent), dtype=np.uint32)[(flags2 & fb.NODE_RENDERABLE) != 0][:3000])
    assert_same_visible(og2, ctx, [fo])
    ctx.build_palettes()
    ctx.skin()
    for u in (0, sc.n_units - 1):
        pos_o, nrm_o = og2.skin(sc.unit_mesh_node(u), 0, sc.verts_per_unit)
        pos_g, nrm_g = ctx.get_skinned(sids[u])
        assert pos_g.tobytes() == pos_o.tobytes() and nrm_g.tobytes() == nrm_o.tobytes()


def test_add_link_remove_then_incremental_update_with_only_the_new_matrices(ctx):
    """The sequence INTEGRATION.md gives the Rust shim (ADVICE r1): fyx_set_topology with the pool's new columns after
    add / link / remove, then upload ONLY the matrices of the new nodes, then an incremental update.  Locals, TRS records,
    transform statics, bundle ids and LOD ranges of the surviving nodes must have followed them to their new slots: the
    result equals an oracle built from scratch with every node's data.  Revived pool records start from the defaults: one
    that is given only a rotation has position 0, scale 1 and the default statics, bundle 0 and no LOD range."""
    from test_gpu_drawprep import check_instances

    rng = np.random.default_rng(17)
    n = 6000
    parent, flags, mask, local, aabb = random_graph(rng, n, p_dead=0.15)
    ctx.set_topology(parent, flags, mask, aabb)
    ctx.set_local_matrices(local)
    # some nodes are driven by TRS records (+ statics): their position / scale live only on the device afterwards
    alive = np.nonzero((flags & fb.NODE_ALIVE) != 0)[0].astype(np.uint32)
    trs_nodes = rng.choice(alive[alive != 0], 400, replace=False).astype(np.uint32)
    trs = np.zeros((len(trs_nodes), 10), np.float32)
    trs[:, 0:3] = rng.uniform(-5, 5, (len(trs_nodes), 3))
    q = rng.normal(size=(len(trs_nodes), 4))
    trs[:, 3:7] = q / np.linalg.norm(q, axis=1, keepdims=True)
    trs[:, 7:10] = rng.uniform(0.5, 2.0, (len(trs_nodes), 3))
    ctx.set_local_trs(trs, trs_nodes)
    eye = (0.0, 0.0, 150.0)  # the whole forest in view
    fo, ff = camera_frustum(eye=eye, target=(0, 0, 0), zfar=800.0, fovy=np.deg2rad(110.0))
    ctx.update_and_cull([ff], fb.UPDATE_ALL)

    # topology B: revive dead pool records as new nodes, re-parent some old nodes, remove some leaves (a removed node takes
    # its sub-tree with it in the reference, so nothing may hang under a removed node)
    dead = np.nonzero((flags & fb.NODE_ALIVE) == 0)[0]
    new_nodes = dead[: len(dead) // 2].astype(np.uint32)
    parent2, flags2, local2 = parent.copy(), flags.copy(), local.copy()
    has_child = np.zeros(n, bool)
    has_child[parent[parent != NONE]] = True
    leaves = alive[(~has_child[alive]) & (alive != 0) & ~np.isin(alive, trs_nodes)]
    removed = leaves[:150]
    flags2[removed] = 0
    survivors = alive[~np.isin(alive, removed)]
    flags2[new_nodes] = fb.NODE_DEFAULT | fb.NODE_RENDERABLE
    parent2[new_nodes] = rng.choice(survivors, len(new_nodes)).astype(np.uint32)
    new_m = np.stack([ob.translation(*rng.uniform(-3, 3, 3)) for _ in new_nodes]).astype(np.float32)
    local2[new_nodes] = new_m
    movers = leaves[150:300]
    parent2[movers] = rng.choice(new_nodes, len(movers)).astype(np.uint32)  # old nodes under the new ones
    # revived records that get nothing but a rotation, under the root
    rng2 = np.random.default_rng(18)
    revived = dead[len(dead) // 2: len(dead) // 2 + 8].astype(np.uint32)
    flags2[revived] = fb.NODE_DEFAULT | fb.NODE_RENDERABLE
    parent2[revived] = 0

    # the side columns, each away from its default, set before topology B
    st_nodes = trs_nodes[:150]
    statics = np.zeros((len(st_nodes), 25), np.float32)
    sq = rng2.normal(size=(len(st_nodes), 4)).astype(np.float32)
    statics[:, 0:4] = sq / np.linalg.norm(sq, axis=1, keepdims=True)
    statics[:, 4:13] = rng2.normal(size=(len(st_nodes), 9)).astype(np.float32)
    statics[:, 13:25] = rng2.uniform(-2, 2, (len(st_nodes), 12)).astype(np.float32)
    ctx.set_transform_statics(statics, st_nodes)
    bundle = rng2.integers(1, 13, n).astype(np.uint32)  # every node; 0 is the default
    ctx.set_bundle_ids(bundle)
    zn, zf = 0.1, 800.0  # the camera's near / far planes, observer at its eye
    # LOD objects: the visible survivors and some others; half of them in range for the observer before topology B
    lod_nodes = np.union1d(np.intersect1d(ctx.get_visible(0), survivors), rng2.choice(survivors[survivors != 0], 200, replace=False))
    lod_nodes = lod_nodes.astype(np.uint32)
    dist = np.linalg.norm(ctx.get_global_matrices(lod_nodes)[:, 12:15] - np.float32(eye), axis=1)
    cut = float(np.median((dist - zn) / (zf - zn)))
    near = rng2.random(len(lod_nodes)) < 0.5
    lod = np.where(near[:, None], [0.0, cut], [cut, 1.0]).astype(np.float32)
    ctx.set_lod_ranges(lod, lod_nodes)
    ctx.set_observers([(eye, zn, zf)])

    ctx.set_topology(parent2, flags2, mask, aabb)
    ctx.set_local_matrices(new_m, new_nodes)  # ONLY the new nodes
    # a rotation-only update of the TRS-driven nodes must still find their positions / scales / statics on the device
    q2 = rng.normal(size=(len(trs_nodes), 4)).astype(np.float32)
    q2 /= np.linalg.norm(q2, axis=1, keepdims=True).astype(np.float32)
    ctx.set_local_rotations(q2, trs_nodes)
    qr = rng2.normal(size=(len(revived), 4)).astype(np.float32)
    qr /= np.linalg.norm(qr, axis=1, keepdims=True).astype(np.float32)
    ctx.set_local_rotations(qr, revived)
    ctx.enable_instances()
    ctx.update_and_cull([ff], fb.UPDATE_INCREMENTAL)

    # the oracle from scratch, with everybody's data
    import sampled_parity as sp

    trs2 = trs.copy()
    trs2[:, 3:7] = q2
    loc = sp.trs_bone_local(trs2)
    for k, i in enumerate(trs_nodes):
        local2[i] = loc(k)
    for k, i in enumerate(st_nodes):
        local2[i] = _oracle_transform(trs2[k, 0:3], trs2[k, 3:7], trs2[k, 7:10], statics[k])
    for k, i in enumerate(revived):
        local2[i] = _oracle_transform(np.zeros(3, np.float32), qr[k], np.ones(3, np.float32))
    og = ob.Graph.build(parent2, flags2, mask, local2, aabb)
    og.L.orc_graph_drop_messages(og.h)
    og.set_lod_group(0, [(float(b), float(e), [int(x)]) for x, (b, e) in zip(lod_nodes, lod)])
    og.update_hierarchical_data()
    # the reference updates what its DFS reaches from the root; orphan sub-trees are not part of the comparison
    live = np.nonzero(reachable_from_root(parent2, flags2))[0].astype(np.uint32)
    assert live.size > 4000 and np.isin(revived, live).all()
    # local rows, TRS records and statics: every reachable node's global transform and box
    assert_same_hierarchy(og, ctx, live)
    # LOD ranges: the culled list is LOD-filtered, and the filter hides something
    want = og.from_graph_lod(fo, eye, zn, zf)
    assert og.from_graph(fo).size - want.size >= 30
    assert np.array_equal(np.sort(ctx.get_visible(0)), np.sort(want))
    # bundle ids: the packed instances of the unfiltered list are grouped by the carried ids, the revived nodes' are 0
    ctx.set_observers([])
    ctx.cull([ff])
    assert_same_visible(og, ctx, [fo])
    bundle2 = bundle.copy()
    bundle2[new_nodes] = 0
    bundle2[revived] = 0
    view = ob.look_at_rh(eye, (0, 0, 0), (0, 1, 0))
    vp = ob.mat4_mul(ob.perspective(16 / 9, float(np.deg2rad(110.0)), zn, zf), view)
    assert check_instances(og, ctx, 0, fo, view, vp, bundle2) > 100
    # removed nodes read back as "not there" (identity / default box), like Pool::try_borrow failing
    assert np.array_equal(ctx.get_global_matrices(removed[:5]), np.tile(np.eye(4, dtype=np.float32).reshape(16), (5, 1)))


def test_dfs_order_quirk_is_reproduced_exactly(ctx):
    """Skinned meshes that come BEFORE (some of) their bones in the reference's DFS: the reference folds those
    bones' positions from before the update (scene/mesh/mod.rs:676-682).  With fyx_set_dfs_order the boxes
    match the oracle's real DFS over several frames, full and incremental updates."""
    rng = np.random.default_rng(33)
    n_units, nb = 40, 12
    # per unit: mesh first, then its bones (chain), all under the root => every bone is "late"; every second unit
    # the other way round (bones first)
    parent, flags, surf = [NONE], [fb.NODE_DEFAULT], []
    for u in range(n_units):
        base = len(parent)
        if u % 2 == 0:
            mesh = base
            parent.append(0)
            flags.append(fb.NODE_DEFAULT | fb.NODE_RENDERABLE)
            bones = list(range(base + 1, base + 1 + nb))
            for k in range(nb):
                parent.append(0 if k == 0 else bones[k - 1])
                flags.append(fb.NODE_DEFAULT)
        else:
            bones = list(range(base, base + nb))
            for k in range(nb):
                parent.append(0 if k == 0 else bones[k - 1])
                flags.append(fb.NODE_DEFAULT)
            mesh = base + nb
            parent.append(0)
            flags.append(fb.NODE_DEFAULT | fb.NODE_RENDERABLE)
        surf.append((mesh, bones))
    parent = np.array(parent, np.uint32)
    flags = np.array(flags, np.uint32)
    n = len(parent)
    aabb = np.tile(UNIT_BOX, (n, 1))

    def random_locals():
        m = np.tile(np.eye(4, dtype=np.float32).reshape(16), (n, 1))
        m[1:, 12:15] = rng.uniform(-6, 6, (n - 1, 3)).astype(np.float32)
        return m

    local = random_locals()
    og = ob.Graph.build(parent, flags, None, local, aabb)
    ctx.set_topology(parent, flags, None, aabb)
    ctx.set_dfs_order(preorder_rank(parent))
    ctx.set_local_matrices(local)
    meshes = np.array([m for m, _ in surf], np.uint32)
    for mesh, bones in surf:
        og.add_surface(mesh, bones)
        ctx.add_skinned_surface(mesh, bones, np.tile(np.eye(4, dtype=np.float32).reshape(16), (nb, 1)))
    og.L.orc_graph_drop_messages(og.h)
    fo, ff = camera_frustum(zfar=400.0)
    for frame in range(4):
        if frame:
            local = random_locals()
            for i in range(1, n):
                og.set_local_matrix(i, local[i])
            ctx.set_local_matrices(local[1:], np.arange(1, n, dtype=np.uint32))
        if frame % 2 == 0:
            og.L.orc_graph_drop_messages(og.h)
            og.update_hierarchical_data()
            ctx.update_and_cull([ff], fb.UPDATE_ALL)
        else:
            # one message root (the scene root): a single DFS, like the full update
            og.L.orc_graph_drop_messages(og.h)
            og.set_local_matrix(0, np.eye(4, dtype=np.float32).reshape(16))
            ctx.set_local_matrices(np.eye(4, dtype=np.float32).reshape(1, 16), [0])
            og.update()
            ctx.update_and_cull([ff], fb.UPDATE_INCREMENTAL)
        assert_same_hierarchy(og, ctx)
        assert_same_visible(og, ctx, [fo])
    # sanity: the quirk is real — without the order the late-bone meshes differ from the reference
    ctx.set_dfs_order(None)
    local = random_locals()
    for i in range(1, n):
        og.set_local_matrix(i, local[i])
    og.L.orc_graph_drop_messages(og.h)
    og.update_hierarchical_data()
    ctx.set_local_matrices(local[1:], np.arange(1, n, dtype=np.uint32))
    ctx.update_transforms(fb.UPDATE_ALL)
    A, Ao = ctx.get_world_aabbs(meshes), og.world_bounding_boxes(meshes)
    early = np.arange(n_units) % 2 == 1
    assert (A[early] == Ao[early]).all() and not (A[~early] == Ao[~early]).all()


def test_k16_reference_vertex_buffer_layout_through_the_c_abi(ctx):
    """tests/golden K16 (fyrox-impl/src/scene/mesh/buffer.rs:1687-1828): the reference's own 76-byte interleaved test vertex handed to
    fyx_add_skinned_surface with a fyx_vertex_layout that names its offsets (position 0, normal 28, bone weights 56, u8 bone indices
    72).  Bones 0..5 translate by (k, 0, 0): every vertex has indices (1, 2, 3, 4) and weights 0.25, so it must come out at
    position + 2.5 on x (exact in f32) with its normal unchanged — the same check the oracle's reader passes on the CPU
    (tests/test_oracle_kat.py::test_k16_...)."""
    import json
    import os

    k = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_kats.json")))["K16_vertex_buffer_attributes"]
    off = k["offsets"]
    nv = len(k["vertices"])
    rec = np.zeros((nv, k["stride"]), np.uint8)
    for i, v in enumerate(k["vertices"]):
        for name in ("position", "tex_coord", "second_tex_coord", "normal", "tangent", "bone_weights"):
            a = np.asarray(v[name], np.float32)
            rec[i, off[name]:off[name] + 4 * a.size] = a.view(np.uint8)
        rec[i, off["bone_indices"]:off["bone_indices"] + 4] = np.asarray(v["bone_indices"], np.uint8)
    nb = 6
    n = nb + 2  # root, six bones, the mesh
    parent = np.array([NONE] + [0] * (n - 1), np.uint32)
    flags = np.full(n, fb.NODE_DEFAULT, np.uint32)
    flags[n - 1] |= fb.NODE_RENDERABLE
    local = np.tile(np.eye(4, dtype=np.float32).reshape(16), (n, 1))
    for b in range(nb):
        local[1 + b, 12] = float(b)
    bones = np.arange(1, nb + 1, dtype=np.uint32)
    ib = np.tile(np.eye(4, dtype=np.float32).reshape(16), (nb, 1))
    ctx.set_topology(parent, flags)
    ctx.set_local_matrices(local)
    layout = fb._lib.fyx_vertex_layout(k["stride"], off["position"], off["normal"], off["bone_weights"], off["bone_indices"])
    sid = ctx.add_skinned_surface(n - 1, bones, ib, rec.reshape(-1), layout=layout)
    ctx.update_transforms(fb.UPDATE_ALL)
    ctx.build_palettes()
    ctx.skin()
    pos, nrm = ctx.get_skinned(sid)
    for i, v in enumerate(k["vertices"]):
        want = np.asarray(v["position"], np.float32) + np.array([2.5, 0.0, 0.0], np.float32)
        assert np.array_equal(pos[i], want), (i, pos[i], want)
        assert np.array_equal(nrm[i], np.asarray(v["normal"], np.float32)), (i, nrm[i])
