"""N3 (SURVEY §8f) — draw-prep after the cull: fyx_pack_instances against the oracle.

Reference: Mesh::collect_render_data (scene/mesh/mod.rs:691-805: sort index, world = identity for skinned
surfaces), RenderDataBundleStorage::push (renderer/bundle.rs:1248-1278: bundle = (material, data, path) key, its
sort index is that of the first instance pushed, i.e. first in DFS order), RenderDataBundle::write_uniforms
(renderer/bundle.rs:483-487: world, view_projection * world).  Bit-exact per instance; order inside a bundle is a set.
"""
import numpy as np
import pytest

import fyrox_b200 as fb
import oracle_binding as ob
from fyrox_b200.scenegen import Scene
from helpers import NONE, bits_equal, cube_frusta, preorder_rank, random_graph, scene_pair

pytestmark = pytest.mark.gpu


def observer(eye, target, up=(0, 1, 0), aspect=16 / 9, fovy=np.deg2rad(60.0), zn=0.1, zf=150.0):
    view = ob.look_at_rh(eye, target, up)
    proj = ob.perspective(float(aspect), float(fovy), float(zn), float(zf))
    vp = ob.mat4_mul(proj, view)  # bundle.rs:894: projection * view
    return view, vp, ob.frustum_from_vp(vp), fb.frustum_from_view_projection_matrix(vp)


def check_instances(og, ctx, f, fo, view, vp, bundle_of_node, rank=None, mask=0xFFFFFFFF, shadow=False):
    inst = ctx.pack_instances(f, view, vp)
    dfs = og.from_graph(fo, mask, shadow)  # the reference's push order
    node = inst["node"]
    assert node.size == dfs.size and np.array_equal(np.sort(node), np.sort(dfs))
    assert np.array_equal(np.sort(node), np.sort(ctx.get_visible(f)))
    # per instance: sort index, world, wvp
    for k in range(node.size):
        si, w, wvp = og.instance(int(node[k]), view, vp)
        assert int(inst["sort_index"][k]) == si, f"sort index of node {node[k]}"
        assert bits_equal(inst["world"][k], w).all(), f"world of node {node[k]}"
        assert bits_equal(inst["wvp"][k], wvp).all(), f"wvp of node {node[k]}"
    # bundle table: ascending ids of the non-empty bundles, a partition of [0, n)
    b = inst["bundles"]
    ids_vis = bundle_of_node[node]
    want_ids = np.unique(ids_vis)
    assert np.array_equal(b["id"], want_ids)
    assert b["first"][0] == 0 if b.size else node.size == 0
    assert np.array_equal(b["first"][1:], np.cumsum(b["count"])[:-1])
    assert int(b["count"].sum()) == node.size
    first_pushed = {}
    if rank is not None:
        for n_ in dfs:  # DFS order: the first instance of each bundle fixes RenderDataBundle::sort_index
            first_pushed.setdefault(int(bundle_of_node[n_]), int(n_))
    for row in b:
        sl = slice(int(row["first"]), int(row["first"] + row["count"]))
        assert (ids_vis[sl] == row["id"]).all(), "an instance sits in the wrong bundle"
        members = node[sl]
        lead = first_pushed[int(row["id"])] if rank is not None else int(members.min())
        assert int(row["sort_index"]) == og.instance(lead, view, vp)[0]
    return node.size


def test_instances_of_generated_scene_match_oracle(ctx):
    sc = Scene(6000, 12)
    og, _ = scene_pair(sc, ctx, with_vertices=False)
    og.update_hierarchical_data()
    rng = np.random.default_rng(5)
    bundle = rng.integers(0, 41, sc.capacity).astype(np.uint32)
    bundle[bundle == 7] = 8  # leave holes in the id space
    ctx.set_bundle_ids(bundle)
    ctx.enable_instances()
    view, vp, fo, ff = observer((3, 2, 25), (0, 0, -10))
    ctx.update_and_cull([ff], fb.UPDATE_ALL)
    n = check_instances(og, ctx, 0, fo, view, vp, bundle)
    assert n > 50
    # skinned meshes among them carry identity
    meshes = {sc.unit_mesh_node(u) for u in range(sc.n_units)}
    inst = ctx.pack_instances(0, view, vp)
    hit = [k for k, nd in enumerate(inst["node"]) if int(nd) in meshes]
    for k in hit:
        assert np.array_equal(inst["world"][k], np.eye(4, dtype=np.float32).reshape(16))
    # stand-alone cull, several frusta, each with its own observer
    obs = [observer((0, 0, 0), (1, 0, 0), (0, -1, 0), 1.0, np.pi / 2, 0.01, 120.0), observer((0, 0, 0), (0, 0, -1)), observer((10, 5, 0), (0, 0, 0))]
    ctx.cull([o[3] for o in obs])
    for f, (v, p, fo_, _) in enumerate(obs):
        check_instances(og, ctx, f, fo_, v, p, bundle)


def test_static_batches_prune_the_dfs_like_rdc_control_flow_break(ctx):
    """A statically batched mesh (BatchingMode::Static) that is rendered for a frustum returns RdcControlFlow::Break: its
    children are not visited FOR THAT FRUSTUM (scene/mesh/mod.rs:701-725, renderer/bundle.rs:996-1001); one that is culled
    lets the DFS continue.  Random forest with static batches at every depth, nested ones, six frusta with masks and a shadow
    pass; fused-capable entry points (they must notice and run the cull un-fused), flags set later through fyx_set_flags."""
    rng = np.random.default_rng(41)
    parent, flags, mask, local, aabb = random_graph(rng, 5000, p_orphan=0.01, max_depth_bias=0.2)
    renderable = np.nonzero((flags & fb.NODE_RENDERABLE) != 0)[0]
    static = rng.choice(renderable, len(renderable) // 6, replace=False)
    flags_s = flags.copy()
    flags_s[static] |= fb.NODE_STATIC_BATCH
    og = ob.Graph.build(parent, flags_s, mask, local, aabb)
    og.L.orc_graph_drop_messages(og.h)
    og.update_hierarchical_data()
    fos, ffs = cube_frusta(radius=200.0)
    cam = np.array([0xFFFFFFFF, 0x0000FFFF, 0xFFFFFFFF, 0xFFFF0000, 0xFFFFFFFF, 0xFFFFFFFF], np.uint32)
    pf = np.array([0, 0, fb.PASS_SHADOW, 0, fb.PASS_SHADOW, 0], np.uint32)
    ctx.set_topology(parent, flags_s, mask, aabb)
    ctx.set_local_matrices(local)
    pruned_something = 0
    for entry in ("update_and_cull", "render_prep", "cull"):
        if entry == "update_and_cull":
            ctx.update_and_cull(ffs, fb.UPDATE_ALL, cam_mask=cam, pass_flags=pf)
        elif entry == "render_prep":
            ctx.render_prep(update_flags=fb.UPDATE_ALL, frusta=ffs, cam_mask=cam, pass_flags=pf)
        else:
            ctx.cull(ffs, cam_mask=cam, pass_flags=pf)
        for f, fo in enumerate(fos):
            want = np.sort(og.from_graph(fo, int(cam[f]), bool(pf[f] & fb.PASS_SHADOW)))
            got = np.sort(ctx.get_visible(f))
            assert np.array_equal(got, want), f"{entry} frustum {f}: {got.size} vs {want.size}"
    # the pruning really happens: without the static flags more nodes are listed
    og0 = ob.Graph.build(parent, flags, mask, local, aabb)
    og0.L.orc_graph_drop_messages(og0.h)
    og0.update_hierarchical_data()
    for f, fo in enumerate(fos):
        pruned_something += og0.from_graph(fo, int(cam[f]), bool(pf[f] & fb.PASS_SHADOW)).size - og.from_graph(fo, int(cam[f]), bool(pf[f] & fb.PASS_SHADOW)).size
    assert pruned_something > 20
    # flags arriving later through fyx_set_flags switch the pruned cull on as well
    with fb.Context() as c2:
        c2.set_topology(parent, flags, mask, aabb)
        c2.set_local_matrices(local)
        c2.update_and_cull(ffs, fb.UPDATE_ALL, cam_mask=cam, pass_flags=pf)
        c2.set_flags(flags_s[static], static.astype(np.uint32))
        c2.update_and_cull(ffs, fb.UPDATE_INCREMENTAL, cam_mask=cam, pass_flags=pf)
        for f, fo in enumerate(fos):
            want = np.sort(og.from_graph(fo, int(cam[f]), bool(pf[f] & fb.PASS_SHADOW)))
            assert np.array_equal(np.sort(c2.get_visible(f)), want)
    # a static batch is pushed with the identity as its world matrix (mesh/mod.rs:716)
    ctx.enable_instances()
    view, vp, fo, ff = observer((0, 0, 0), (0, 0, -1), zf=400.0, fovy=np.deg2rad(120.0))
    ctx.update_and_cull([ff], fb.UPDATE_ALL)
    inst = ctx.pack_instances(0, view, vp)
    st = set(int(x) for x in static)
    seen = 0
    for k, nd in enumerate(inst["node"]):
        si, w, wvp = og.instance(int(nd), view, vp)
        assert inst["world"][k].tobytes() == w.tobytes() and inst["wvp"][k].tobytes() == wvp.tobytes()
        if int(nd) in st:
            assert np.array_equal(inst["world"][k], np.eye(4, dtype=np.float32).reshape(16))
            seen += 1
    assert seen > 0


def test_meshes_with_several_surfaces_push_one_instance_per_surface(ctx):
    """Mesh::collect_render_data pushes one SurfaceInstanceData per surface (scene/mesh/mod.rs:726-805): each goes to the
    bundle of its own key, carries the identity if IT is skinned and the node's global transform otherwise, its own bone
    matrices, and the node's sort index.  Skinned units get 3 surfaces (skinned, static, skinned with other bones), some
    static leaves 2; everybody else keeps the default single surface."""
    import ctypes as C

    sc = Scene(5000, 10, verts_per_unit=64)
    og, sids = scene_pair(sc, ctx)
    idx, m = sc.animate(1)
    for i, mm in zip(idx, m):
        og.set_local_matrix(int(i), mm)
    og.update_hierarchical_data()
    rng = np.random.default_rng(8)
    bundle = rng.integers(0, 23, sc.capacity).astype(np.uint32)  # default (single-surface) bundle ids
    ctx.set_bundle_ids(bundle)
    nodes, surfaces, want_key = [], [], {}
    for u in range(sc.n_units):
        mesh = int(sc.unit_mesh_node(u))
        bones = sc.unit_bone_nodes(u)
        # oracle: surface 0 exists (all bones); add an unskinned one and one skinned by the first 5 bones
        og.add_surface(mesh, np.empty(0, np.uint32))
        og.add_surface(mesh, bones[:5])
        sid2 = ctx.add_skinned_surface(mesh, bones[:5], sc.unit_inv_bind(u)[:5], None, n_verts=0)
        lst = [(int(rng.integers(30, 40)), sids[u]), (int(rng.integers(30, 40)), None), (int(rng.integers(30, 40)), sid2)]
        nodes.append(mesh)
        surfaces.append(lst)
        for k, (bid, _) in enumerate(lst):
            want_key[(mesh, k)] = bid
    leaves = np.nonzero((sc.flags & fb.NODE_RENDERABLE) != 0)[0]
    for leaf in leaves[:200:2]:
        leaf = int(leaf)
        if leaf in nodes:
            continue
        og.add_surface(leaf, np.empty(0, np.uint32))
        og.add_surface(leaf, np.empty(0, np.uint32))
        lst = [(int(rng.integers(40, 45)), None), (int(rng.integers(40, 45)), None)]
        nodes.append(leaf)
        surfaces.append(lst)
        for k, (bid, _) in enumerate(lst):
            want_key[(leaf, k)] = bid
    ctx.set_node_surfaces(nodes, surfaces)
    ctx.enable_instances()
    view, vp, fo, ff = observer((0, 0, 400), (0, 0, 0), zf=900.0)
    ctx.render_prep(update_flags=fb.UPDATE_ALL, changed_m16=m, changed_idx=idx, frusta=[ff])
    inst = ctx.pack_instances(0, view, vp)
    ctx.pack_bone_matrices(0)
    vis = og.from_graph(fo)
    multi = {n_: len(l) for n_, l in zip(nodes, surfaces)}
    assert inst["node"].size == sum(multi.get(int(n_), 1) for n_ in vis)
    L = ob.lib()
    seen = set()
    b = inst["bundles"]
    owner = np.empty(inst["node"].size, np.uint32)
    for row in b:
        owner[int(row["first"]): int(row["first"] + row["count"])] = row["id"]
    n_multi = n_blocks = 0
    for k in range(inst["node"].size):
        nd, sf = int(inst["node"][k]), int(inst["surface"][k])
        assert (nd, sf) not in seen
        seen.add((nd, sf))
        blk = ctx.get_bone_matrix_block(0, k)
        want = np.empty(255 * 16, np.float32)
        if nd in multi:
            w = np.empty(16, np.float32)
            wvp = np.empty(16, np.float32)
            sk = C.c_int()
            # the oracle's surface ordinals of a unit mesh: 0 = the scene's skinned surface, 1, 2 = the two added above
            si = L.orc_node_surface_instance(og.h, nd, sf, ob.fp(np.ascontiguousarray(view)), ob.fp(np.ascontiguousarray(vp)), ob.fp(w), ob.fp(wvp), C.byref(sk))
            has = L.orc_surface_bone_block(og.h, nd, sf, ob.fp(want))
            assert bool(has) == bool(sk.value)
        else:  # the default: one surface, as Mesh::collect_render_data treats a single-surface mesh
            assert sf == 0
            si, w, wvp = og.instance(nd, view, vp)
            has = L.orc_instance_bone_block(og.h, nd, ob.fp(want))
        assert int(inst["sort_index"][k]) == si
        assert inst["world"][k].tobytes() == w.tobytes() and inst["wvp"][k].tobytes() == wvp.tobytes()
        assert int(owner[k]) == want_key.get((nd, sf), int(bundle[nd]))
        assert bool(has) == (blk is not None)
        if has:
            assert blk.reshape(-1).tobytes() == want.tobytes()
            n_blocks += 1
        n_multi += nd in multi
    assert n_multi > 30 and n_blocks >= 6
    # every (visible node, surface) pair is there
    assert seen == {(int(n_), k) for n_ in vis for k in range(multi.get(int(n_), 1))}


def test_bone_matrix_blocks_of_packed_instances_match_oracle(ctx):
    """N3: every skinned instance of the packed list carries the 255-mat4 block write_uniforms builds (bone_matrices, then
    zero matrices, renderer/bundle.rs:484-496); unskinned instances carry none."""
    sc = Scene(6000, 14, verts_per_unit=64)
    og, sids = scene_pair(sc, ctx)
    idx, m = sc.animate(1)
    for i, mm in zip(idx, m):
        og.set_local_matrix(int(i), mm)
    og.update_hierarchical_data()
    ctx.enable_instances()
    view, vp, fo, ff = observer((0, 0, 400), (0, 0, 0), zf=900.0)  # far enough back to see the whole scene
    ctx.render_prep(update_flags=fb.UPDATE_ALL, changed_m16=m, changed_idx=idx, frusta=[ff])
    inst = ctx.pack_instances(0, view, vp)
    ctx.pack_bone_matrices(0)
    meshes = {int(sc.unit_mesh_node(u)) for u in range(sc.n_units)}
    L = ob.lib()
    seen = 0
    for k, nd in enumerate(inst["node"]):
        blk = ctx.get_bone_matrix_block(0, k)
        want = np.empty(255 * 16, np.float32)
        has = L.orc_instance_bone_block(og.h, int(nd), ob.fp(want))
        assert bool(has) == (int(nd) in meshes) == (blk is not None)
        if has:
            assert blk.reshape(-1).tobytes() == want.tobytes()
            assert not blk[sc.bones_per_unit:].any()
            seen += 1
    assert seen >= 3  # several skinned meshes are in view


def test_bundle_sort_index_follows_the_dfs_push_order(ctx):
    rng = np.random.default_rng(77)
    parent, flags, mask, local, aabb = random_graph(rng, 3000, p_orphan=0.02)
    og = ob.Graph.build(parent, flags, mask, local, aabb)
    og.update_hierarchical_data()
    ctx.set_topology(parent, flags, mask, aabb)
    rank = preorder_rank(parent)
    ctx.set_dfs_order(rank)
    ctx.set_local_matrices(local)
    bundle = rng.integers(0, 9, len(parent)).astype(np.uint32)
    ctx.set_bundle_ids(bundle)
    ctx.enable_instances()
    view, vp, fo, ff = observer((0, 0, 60), (0, 0, 0), zf=200.0)
    ctx.update_and_cull([ff], fb.UPDATE_ALL)
    assert check_instances(og, ctx, 0, fo, view, vp, bundle, rank=rank) > 20
    # index-shuffled forest: the first-pushed instance is generally NOT the lowest node index
    dfs = og.from_graph(fo)
    differs = 0
    for b_ in np.unique(bundle[dfs]):
        m = dfs[bundle[dfs] == b_]
        differs += int(m[0] != m.min())
    assert differs > 0
    # shadow pass + camera mask go through the same lists
    ctx.cull([ff], cam_mask=[0x0000FFFF], pass_flags=[fb.PASS_SHADOW])
    check_instances(og, ctx, 0, fo, view, vp, bundle, rank=rank, mask=0x0000FFFF, shadow=True)


def test_instances_edge_cases(ctx):
    # default bundle (no ids given), empty visible list, projective / degenerate view matrices, errors
    sc = Scene(800, 2)
    og, _ = scene_pair(sc, ctx, with_vertices=False)
    og.update_hierarchical_data()
    view, vp, fo, ff = observer((0, 0, 0), (0, 0, -1))
    ctx.update_and_cull([ff], fb.UPDATE_ALL)
    with pytest.raises(fb.FyxError):
        ctx.pack_instances(0, view, vp)  # cull made without enable_instances
    ctx.enable_instances()
    ctx.cull([ff])
    zeros = np.zeros(sc.capacity, np.uint32)
    check_instances(og, ctx, 0, fo, view, vp, zeros)
    with pytest.raises(fb.FyxError):
        ctx.pack_instances(3, view, vp)
    # a view matrix with a projective bottom row and one whose n is 0 for some points (transform_point skips the divide)
    weird = view.copy()
    weird[3], weird[7], weird[11], weird[15] = 0.01, -0.02, 0.005, 0.0
    check_instances(og, ctx, 0, fo, weird, vp, zeros)
    huge = view.copy() * np.float32(1e30)  # sort index saturates at both ends / NaN -> centre
    check_instances(og, ctx, 0, fo, huge, vp, zeros)
    # a frustum far away from everything: only the nodes with frustum culling switched off remain
    _, _, fo2, ff2 = observer((0, 5000, 0), (0, 6000, 0), (1, 0, 0))
    ctx.cull([ff2])
    assert check_instances(og, ctx, 0, fo2, view, vp, zeros) < 50
    # nothing visible at all (no render-mask bit in common)
    ctx.cull([ff2], cam_mask=[0])
    inst = ctx.pack_instances(0, view, vp)
    assert inst["node"].size == 0 and inst["bundles"].size == 0
    # ids must be dense
    with pytest.raises(fb.FyxError):
        ctx.set_bundle_ids(np.array([1 << 30], np.uint32), [1])


def test_light_lists_match_oracle(ctx):
    """N4 (light list): the collect_lights loop of from_graph (renderer/bundle.rs:926-974) — lights are tested against the
    frustum by their world box and by global visibility / enabled only; lights with frustum culling switched off and
    lights whose render mask misses the camera's still follow exactly that rule.  (Sub-trees detached from the root are
    left out: the reference never updates them, so a light in one is tested with whatever its last update left.)"""
    rng = np.random.default_rng(909)
    parent, flags, mask, local, aabb = random_graph(rng, 4000, p_orphan=0.0, p_mesh=0.5)
    alive = (flags & fb.NODE_ALIVE) != 0
    pivots = alive & ((flags & fb.NODE_RENDERABLE) == 0)
    lights = pivots & (rng.random(len(flags)) < 0.3)
    lights[0] = False
    flags = flags.copy()
    flags[lights] |= fb.NODE_LIGHT
    og = ob.Graph.build(parent, flags, mask, local, aabb)
    og.update_hierarchical_data()
    ctx.set_topology(parent, flags, mask, aabb)
    ctx.set_local_matrices(local)
    with pytest.raises(fb.FyxError):
        ctx.cull_lights()  # no cull yet
    obs = [observer((0, 0, 60), (0, 0, 0), zf=200.0), observer((0, 0, 0), (1, 0, 0), (0, -1, 0), 1.0, np.pi / 2, 0.01, 120.0),
           observer((30, 10, -20), (0, 0, 0), zf=80.0)]
    ctx.update_and_cull([o[3] for o in obs], fb.UPDATE_ALL, cam_mask=[0xFFFFFFFF, 0x0000FFFF, 0xFFFFFFFF])
    ctx.cull_lights()
    total = 0
    for f, o in enumerate(obs):
        want = og.collect_lights(o[2])
        got = ctx.get_visible_lights(f)
        assert np.array_equal(got, want)  # same set AND the reference's pool order
        total += want.size
    assert total > 30
    # a light switched off by an ancestor's visibility disappears; flags can change at run time
    some = np.nonzero(lights)[0][:40].astype(np.uint32)
    newf = flags[some] & ~np.uint32(fb.NODE_ENABLED)
    for i in some:
        ob.lib().orc_node_set_enabled(og.h, int(i), 0)
    og.update()
    ctx.set_flags(newf, some)
    ctx.update_and_cull([o[3] for o in obs], fb.UPDATE_INCREMENTAL)
    ctx.cull_lights()
    for f, o in enumerate(obs):
        assert np.array_equal(ctx.get_visible_lights(f), og.collect_lights(o[2]))


def test_reflection_probe_selection_matches_oracle(ctx):
    """The reflection-probe part of from_graph's node loop (renderer/bundle.rs:918-925): the LAST probe in pool order whose world
    box contains the observer wins; no probe -> none; boxes that only touch the observer count (inclusive compares)."""
    rng = np.random.default_rng(23)
    parent, flags, mask, local, aabb = random_graph(rng, 3000, p_orphan=0.0)
    # probes among the nodes whose box the oracle takes from the caller as well (its pivots keep Base's unit box)
    alive = np.nonzero((flags & fb.NODE_ALIVE) != 0)[0]
    alive = alive[(flags[alive] & fb.NODE_RENDERABLE) != 0]
    probes = rng.choice(alive[alive != 0], 60, replace=False)
    flags = flags.copy()
    flags[probes] |= fb.NODE_REFLECTION_PROBE
    aabb = aabb.copy()
    h = rng.uniform(5.0, 40.0, (len(probes), 3)).astype(np.float32)  # big boxes: several contain a given point
    aabb[probes, :3], aabb[probes, 3:] = -h, h
    og = ob.Graph.build(parent, flags, mask, local, aabb)
    og.L.orc_graph_drop_messages(og.h)
    og.update_hierarchical_data()
    ctx.set_topology(parent, flags, mask, aabb)
    ctx.set_local_matrices(local)
    ctx.update_transforms(fb.UPDATE_ALL)
    # observers: random points, the centre of a probe's box, a point exactly ON a probe's box face, far away
    reach = [int(p) for p in probes]
    boxes = ctx.get_world_aabbs(np.array(reach, np.uint32))
    obs = [tuple(rng.uniform(-30, 30, 3).astype(np.float32)) for _ in range(4)]
    obs.append(tuple(((boxes[0, :3] + boxes[0, 3:]) * np.float32(0.5)).astype(np.float32)))
    obs.append((float(boxes[1, 3]), float(boxes[1, 1] + boxes[1, 4]) * 0.5, float(boxes[1, 2] + boxes[1, 5]) * 0.5))  # on the +x face
    obs.append((1e6, 1e6, 1e6))
    ctx.set_observers([(o, 0.1, 100.0) for o in obs])
    got = ctx.select_reflection_probes()
    hits = 0
    for k, o in enumerate(obs):
        want = og.L.orc_select_reflection_probe(og.h, ob.fp(np.array(o, np.float32)))
        assert int(got[k]) == int(want), (k, o, got[k], want)
        hits += want != NONE
    assert int(got[-1]) == NONE and hits >= 3
    ctx.set_observers([])


def test_lod_filter_matches_oracle(ctx):
    """N4 (LOD filter): from_graph's lod_filter (renderer/bundle.rs:898-916) and the pruned DFS (:988-1004) — a LOD object
    outside its level's normalised-distance range hides its whole sub-tree for that observer; objects listed by several
    owners take the verdict written last; fused, stand-alone and one-call culls; switching the filter off again."""
    rng = np.random.default_rng(1234)
    parent, flags, mask, local, aabb = random_graph(rng, 3000, p_orphan=0.02, p_mesh=0.7)
    n = len(parent)
    og = ob.Graph.build(parent, flags, mask, local, aabb)
    og.update_hierarchical_data()
    ctx.set_topology(parent, flags, mask, aabb)
    ctx.set_local_matrices(local)
    alive = np.nonzero((flags & fb.NODE_ALIVE) != 0)[0]
    owners = np.sort(rng.choice(alive, 30, replace=False))
    levels = [(0.0, 0.25), (0.25, 0.6), (0.6, 1.0)]
    final = {}
    for o in owners:  # pool order, levels in order, objects in order: the last write wins (what the host resolves)
        lv = []
        for (b, e) in levels:
            objs = rng.integers(1, n, rng.integers(1, 5)).tolist()  # may hit dead records and other owners' objects
            lv.append((b, e, objs))
            for x in objs:
                if flags[x] & fb.NODE_ALIVE:
                    final[x] = (b, e)
        og.set_lod_group(int(o), lv)
    idx = np.array(sorted(final), np.uint32)
    ctx.set_lod_ranges(np.array([final[int(i)] for i in idx], np.float32), idx)
    eyes = [((0, 0, 60), (0, 0, 0), 0.1, 200.0), ((35, 5, -10), (0, 0, 0), 0.5, 90.0), ((-20, -30, 15), (5, 5, 5), 0.1, 60.0)]
    obs = [observer(e, t, zn=zn, zf=zf) for e, t, zn, zf in eyes]
    observers = [(e, zn, zf) for e, _, zn, zf in eyes]
    ffs = [o[3] for o in obs]

    def check(lod=True):
        hidden = 0
        for f, (e, _, zn, zf) in enumerate(eyes):
            plain = og.from_graph(obs[f][2])
            want = og.from_graph_lod(obs[f][2], e, zn, zf) if lod else plain
            got = np.sort(ctx.get_visible(f))
            assert np.array_equal(got, np.sort(want)), f"frustum {f}: {got.size} vs {want.size}"
            hidden += plain.size - want.size
        return hidden

    ctx.update_and_cull(ffs, fb.UPDATE_ALL)
    assert check(lod=False) == 0  # ranges alone do nothing: no observers yet
    ctx.set_observers(observers)
    ctx.update_and_cull(ffs, fb.UPDATE_ALL)
    assert check() > 20  # the filter really removes nodes
    ctx.cull(ffs)
    check()
    ctx.render_prep(update_flags=fb.UPDATE_INCREMENTAL, frusta=ffs, do_palettes=False, do_skin=False)
    check()
    # a cull with another frustum count is not LOD-filtered (the observers do not match it)
    ctx.cull(ffs[:2])
    for f in range(2):
        assert np.array_equal(np.sort(ctx.get_visible(f)), np.sort(og.from_graph(obs[f][2])))
    # remove half of the objects from LOD control, move the graph, cull again
    drop = idx[::2]
    ctx.set_lod_ranges(np.full((drop.size, 2), np.nan, np.float32), drop)
    dropped = set(int(x) for x in drop)
    for o in owners:
        og.set_lod_group(int(o), [])
    # rebuild the oracle's groups from what is left: one single-object level per remaining object keeps the same verdicts
    rest = [int(i) for i in idx if int(i) not in dropped]
    for k, x in enumerate(rest):
        og.set_lod_group(int(owners[k % len(owners)]), [])
    per_owner = {}
    for k, x in enumerate(rest):
        per_owner.setdefault(int(owners[k % len(owners)]), []).append((final[x][0], final[x][1], [x]))
    for o, lv in per_owner.items():
        og.set_lod_group(o, lv)
    ctx.update_and_cull(ffs, fb.UPDATE_ALL)
    check()
    ctx.set_observers([])
    ctx.cull(ffs)
    assert check(lod=False) == 0
