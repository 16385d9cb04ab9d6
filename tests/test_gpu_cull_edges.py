"""Every device frustum-box test held to the reference loop on boxes that sit on the rounding edge (tests/cull_edges.py).

The kernels' predicate (fyx_math.cuh, frustum_intersects_aabb) replaces Frustum::is_intersects_aabb's 8 corners x 6 planes loop
with a max corner per plane, a reject against pm, a fallback over distinct corner coordinates and a per-lane literal path for
non-tame boxes, and it is compiled into many separate kernels.  Each case here runs one of them on edge boxes and compares
twice: the visible sets with the oracle, and every node's decision with cull_edges.literal_intersects on the world box the
device read back.  A census of the decisions per edge class asserts that each case still reaches the edges."""
import os
import subprocess
import sys

import numpy as np
import pytest

import cull_edges as ce
import fyrox_b200 as fb
import oracle_binding as ob
from helpers import NONE, UNIT_BOX, bits_equal

pytestmark = pytest.mark.gpu
f32 = np.float32
RENDER = fb.NODE_DEFAULT | fb.NODE_RENDERABLE
HERE = os.path.dirname(os.path.abspath(__file__))
IDENTITY = np.eye(4, dtype=f32).reshape(16)
# decisions per class a case must reach (over all its frusta); the fallback classes are the ones only a corner decides
MIN_CENSUS = {"plane_zero": 4, "plane_above": 4, "plane_below": 4, "pm_equal": 4, "pm_below": 2, "corner_on": 8, "corner_in": 8,
              "corner_out": 8, "single_corner": 4, "point_plane": 1, "point_corner": 2, "non_tame": 4, "fallback": 4, "fallback_true": 2}


def pick_frusta(rng, n):
    """n of the eight edge shapes, starting at a different one for each count so that every shape meets several NFT forms."""
    fr = ce.edge_frusta(rng)
    return [fr[(n + i) % len(fr)] for i in range(n)]


def masks_for(n_frusta):
    """Camera masks and shadow passes mixed in: frustum 1 sees only the low 16 mask bits, frustum 2 is a shadow pass."""
    cam = np.full(n_frusta, 0xFFFFFFFF, np.uint32)
    pf = np.zeros(n_frusta, np.uint32)
    if n_frusta > 1:
        cam[1] = 0x0000FFFF
    if n_frusta > 2:
        pf[2] = fb.PASS_SHADOW
    return cam, pf


def flat_scene(boxes, rng):
    """Root 0 with one renderable child per box, identity local matrices (the world box is the local box, -0 aside)."""
    n = len(boxes) + 1
    parent = np.zeros(n, np.uint32)
    parent[0] = NONE
    flags = np.full(n, RENDER, np.uint32)
    flags[0] = fb.NODE_DEFAULT
    flags[1:] &= ~np.where(rng.random(n - 1) < 0.25, fb.NODE_CAST_SHADOWS, 0).astype(np.uint32)
    mask = np.where(rng.random(n) < 0.8, 0xFFFFFFFF, 1 << rng.integers(0, 32, n)).astype(np.uint32)
    local = np.tile(IDENTITY, (n, 1))
    aabb = np.concatenate([UNIT_BOX[None], boxes]).astype(f32)
    return parent, flags, mask, local, aabb


def load(ctx, parent, flags, mask, local, aabb):
    og = ob.Graph.build(parent, flags, mask, local, aabb)
    og.update_hierarchical_data()
    ctx.set_topology(parent, flags, mask, aabb)
    ctx.set_local_matrices(local)
    return og


def check_visible(og, ctx, frusta, nodes, flags, mask, cam, pf, census, got_of=None, want_of=None):
    """Visible sets against the oracle, and each of `nodes`' decisions against the literal loop on its read-back world box."""
    W = ctx.get_world_aabbs(nodes)
    assert bits_equal(W, og.world_bounding_boxes(nodes)).all()
    for f, ef in enumerate(frusta):
        shadow = bool(pf[f] & fb.PASS_SHADOW)
        got = np.sort(ctx.get_visible(f) if got_of is None else got_of(f))
        want = np.sort(og.from_graph(ef.fo, int(cam[f]), shadow) if want_of is None else want_of(f))
        assert got.size == np.unique(got).size
        assert np.array_equal(got, want), (ef.name, f, got.size, want.size)
        eligible = ((mask[nodes] & cam[f]) != 0) & ((not shadow) | ((flags[nodes] & fb.NODE_CAST_SHADOWS) != 0))
        lit = ef.intersects(W)
        mine = np.isin(nodes, got)
        bad = mine != (eligible & lit)
        assert not bad.any(), (ef.name, f, nodes[bad][:5], W[bad][:3], lit[bad][:5])
        for c, m in ce.classify(ef.planes, ef.corners, W[eligible]).items():
            census[c] = census.get(c, 0) + int(m.sum())


def assert_census(census, scale=1, frusta=()):
    """Minimum decisions per class; where a frustum has more than four distinct corner coordinates on an axis (the rotated
    perspectives, the maps' frusta), the fallback must also have been decided by the second half of those lists."""
    want = dict(MIN_CENSUS)
    if any(max(len(np.unique(ef.corners[:, k].view(np.uint32))) for k in range(3)) > 4 for ef in frusta):
        want["fallback_late_coord"] = 1
    short = {c: census.get(c, 0) for c, k in want.items() if census.get(c, 0) < k * scale}
    assert not short, (short, census)
    print("census", census)


# ---- 1. fused fyx_update_and_cull: k_update_level<NFT, UA> --------------------------------------------------------------------
@pytest.mark.parametrize("update", ["all", "incremental"])
@pytest.mark.parametrize("n_frusta", [1, 2, 3, 4, 5, 6, 7, 8])
def test_fused_update_and_cull_on_edge_boxes(ctx, n_frusta, update):
    rng = np.random.default_rng(100 + n_frusta)
    frusta = pick_frusta(rng, n_frusta)
    cam, pf = masks_for(n_frusta)
    parent, flags, mask, local, aabb = flat_scene(ce.all_boxes(frusta, rng), rng)
    nodes = np.arange(1, len(parent), dtype=np.uint32)
    census = {}
    og = load(ctx, parent, flags, mask, local, aabb)
    ctx.update_and_cull([ef.ff for ef in frusta], fb.UPDATE_ALL, cam, pf)
    check_visible(og, ctx, frusta, nodes, flags, mask, cam, pf, census)
    if update == "incremental":
        # new edge boxes for the same nodes, every local matrix sent again: the incremental form recomputes and culls them all
        aabb2 = np.concatenate([UNIT_BOX[None], ce.all_boxes(frusta, rng)[:len(nodes)]]).astype(f32)
        if len(aabb2) < len(aabb):
            aabb2 = np.concatenate([aabb2, aabb[len(aabb2):]])
        og = ob.Graph.build(parent, flags, mask, local, aabb2)
        og.update_hierarchical_data()
        ctx.set_local_aabbs(aabb2)
        ctx.set_local_matrices(local)
        ctx.update_and_cull([ef.ff for ef in frusta], fb.UPDATE_INCREMENTAL, cam, pf)
        check_visible(og, ctx, frusta, nodes, flags, mask, cam, pf, census)
    assert_census(census, frusta=frusta)


# ---- 2. stand-alone fyx_cull: k_cull<NFT>, flat and masked by the camera's pruner table ---------------------------------------
@pytest.mark.parametrize("n_frusta", [1, 2, 3, 4, 5, 6, 7, 8])
def test_cull_on_edge_boxes(ctx, n_frusta):
    rng = np.random.default_rng(200 + n_frusta)
    frusta = pick_frusta(rng, n_frusta)
    cam, pf = masks_for(n_frusta)
    parent, flags, mask, local, aabb = flat_scene(ce.all_boxes(frusta, rng), rng)
    og = load(ctx, parent, flags, mask, local, aabb)
    ctx.update_transforms(fb.UPDATE_ALL)
    ctx.cull([ef.ff for ef in frusta], cam, pf)
    census = {}
    check_visible(og, ctx, frusta, np.arange(1, len(parent), dtype=np.uint32), flags, mask, cam, pf, census)
    assert_census(census, frusta=frusta)


@pytest.mark.parametrize("n_frusta", [1, 3, 6, 7])
def test_cull_with_static_batch_and_lod_group_on_edge_boxes(ctx, n_frusta):
    """A static batch (its sub-tree is pruned where the batch is visible) and LOD objects (hidden where out of range) make k_cull
    run after the camera's pruner table; the edge boxes hang under the batch, on the LOD objects and beside them."""
    rng = np.random.default_rng(300 + n_frusta)
    frusta = pick_frusta(rng, n_frusta)
    cam, pf = masks_for(n_frusta)
    boxes = ce.all_boxes(frusta, rng)
    m = len(boxes)
    parent, flags, mask, local, aabb = flat_scene(boxes, rng)
    # node 1 becomes the static batch: a box around everything, its children the first quarter of the edge boxes
    batch = 1
    aabb[batch] = (-1e6, -1e6, -1e6, 1e6, 1e6, 1e6)
    flags[batch] |= fb.NODE_STATIC_BATCH | fb.NODE_CAST_SHADOWS
    mask[batch] = 0xFFFFFFFF
    under = np.arange(2, 2 + m // 4, dtype=np.uint32)
    parent[under] = batch
    # the next quarter are LOD objects, half of them out of range
    lod_nodes = np.arange(2 + m // 4, 2 + m // 2, dtype=np.uint32)
    ranges = np.where((rng.random(len(lod_nodes)) < 0.5)[:, None], [0.0, 1.0], [0.999, 1.0]).astype(f32)
    og = ob.Graph.build(parent, flags, mask, local, aabb)
    og.L.orc_graph_drop_messages(og.h)
    og.set_lod_group(0, [(float(b), float(e), [int(x)]) for x, (b, e) in zip(lod_nodes, ranges)])
    og.update_hierarchical_data()
    ctx.set_topology(parent, flags, mask, aabb)
    ctx.set_local_matrices(local)
    ctx.set_lod_ranges(ranges, lod_nodes)
    eye, zn, zf = np.array([3.0, -2.0, 7.0], f32), 0.1, 150.0
    ctx.set_observers([(eye, zn, zf)] * n_frusta)
    ctx.update_transforms(fb.UPDATE_ALL)
    ctx.cull([ef.ff for ef in frusta], cam, pf)
    census = {}
    free = np.arange(2 + m // 2, len(parent), dtype=np.uint32)  # neither pruned nor filtered: decided by the predicate alone
    want_of = lambda f: og.from_graph_lod(frusta[f].fo, eye, zn, zf, int(cam[f]), bool(pf[f] & fb.PASS_SHADOW))
    check_visible(og, ctx, frusta, free, flags, mask, cam, pf, census, want_of=want_of)
    # the LOD objects in range and the batch's children where the batch is not visible follow the predicate too
    W = ctx.get_world_aabbs(np.concatenate([under, lod_nodes]))
    # every LOD object has an identity local matrix: it sits at the origin, at a normalized distance of ~0.05 from the observer,
    # inside the range [0, 1] and outside [0.999, 1] — the expectation below rests on that
    d = (np.linalg.norm(eye.astype(np.float64)) - zn) / (zf - zn)
    assert 0.0 <= d < 0.999 and (ctx.get_global_matrices(lod_nodes)[:, 12:15] == 0).all()
    hidden_somewhere = 0
    for f, ef in enumerate(frusta):
        got = ctx.get_visible(f)
        shadow = bool(pf[f] & fb.PASS_SHADOW)
        batch_vis = batch in got
        lit = ef.intersects(W)
        both = np.concatenate([under, lod_nodes])
        eligible = ((mask[both] & cam[f]) != 0) & ((not shadow) | ((flags[both] & fb.NODE_CAST_SHADOWS) != 0))
        expect = eligible & lit
        expect[:len(under)] &= not batch_vis
        expect[len(under):] &= ranges[:, 0] == 0.0
        assert np.array_equal(np.isin(both, got), expect), ef.name
        hidden_somewhere += int((eligible & lit & ~expect).sum())
    assert hidden_somewhere > 0
    ctx.set_observers([])
    assert_census(census, frusta=frusta)


# ---- 3. deep narrow chains: k_update_subforest<{1,6,0}> or one launch per level ----------------------------------------------
@pytest.mark.parametrize("n_frusta", [1, 5, 6])
def test_deep_chains_with_edge_boxes_on_the_deep_levels(ctx, n_frusta):
    rng = np.random.default_rng(400 + n_frusta)
    frusta = pick_frusta(rng, n_frusta)
    cam, pf = masks_for(n_frusta)
    boxes = ce.all_boxes(frusta, rng)
    n_chains, top = 24, 6  # 24 nodes per level; the first `top` levels carry plain boxes
    depth = top + -(-len(boxes) // n_chains)
    n = 1 + n_chains * depth
    parent = np.empty(n, np.uint32)
    parent[0] = NONE
    ids = 1 + np.arange(n_chains * depth).reshape(depth, n_chains)  # level-major: node ids[l, c]
    parent[ids[0]] = 0
    parent[ids[1:]] = ids[:-1]
    flags = np.full(n, RENDER, np.uint32)
    flags[0] = fb.NODE_DEFAULT
    flags[1:] &= ~np.where(rng.random(n - 1) < 0.25, fb.NODE_CAST_SHADOWS, 0).astype(np.uint32)
    mask = np.where(rng.random(n) < 0.8, 0xFFFFFFFF, 1 << rng.integers(0, 32, n)).astype(np.uint32)
    local = np.tile(IDENTITY, (n, 1))
    aabb = np.tile(UNIT_BOX, (n, 1))
    deep = ids[top:].reshape(-1)
    aabb[deep[:len(boxes)]] = boxes
    census = {}
    for update in (fb.UPDATE_ALL, fb.UPDATE_INCREMENTAL):
        og = load(ctx, parent, flags, mask, local, aabb)
        ctx.update_and_cull([ef.ff for ef in frusta], update, cam, pf)
        check_visible(og, ctx, frusta, deep[:len(boxes)].astype(np.uint32), flags, mask, cam, pf, census)
    assert_census(census, frusta=frusta)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("mode", ["0", "1"])
def test_deep_chains_with_the_subforest_kernel_forced(mode):
    """FYX_SUBFOREST=1 / =0 (read when the library first launches it): the same chains through k_update_subforest or one launch
    per level, each in its own process."""
    e = dict(os.environ)
    e["FYX_SUBFOREST"] = mode
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", "-k", "deep_chains_with_edge_boxes",
                        os.path.join(HERE, "test_gpu_cull_edges.py")], capture_output=True, text=True, env=e, timeout=850)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert "3 passed" in r.stdout


# ---- 4. skinned meshes: k_fold_bones<{1,6,0}> culls in lanes 0-7 of warp 0 ----------------------------------------------------
@pytest.mark.parametrize("n_frusta", [1, 6, 5])
def test_skinned_meshes_folded_onto_edge_boxes(ctx, n_frusta):
    """Each mesh has two bones, at the min and the max corner of an edge box, and a local box that is a point at the first bone:
    the folded world box is the edge box.  8 meshes per CTA (one per warp), several CTAs and a partly filled last one."""
    rng = np.random.default_rng(500 + n_frusta)
    frusta = pick_frusta(rng, n_frusta)
    cam, pf = masks_for(n_frusta)
    boxes = ce.all_boxes(frusta, rng)
    finite = np.isfinite(boxes).all(1) & (boxes[:, :3] <= boxes[:, 3:]).all(1)
    boxes = boxes[finite][: 8 * 37 + 5]
    k = len(boxes)
    n = 1 + 3 * k
    parent = np.zeros(n, np.uint32)
    parent[0] = NONE
    flags = np.full(n, fb.NODE_DEFAULT, np.uint32)
    mesh = 3 + 3 * np.arange(k, dtype=np.uint32)  # bones mesh-2, mesh-1 come first in the DFS
    flags[mesh] |= fb.NODE_RENDERABLE
    flags[mesh] &= ~np.where(rng.random(k) < 0.25, fb.NODE_CAST_SHADOWS, 0).astype(np.uint32)
    mask = np.where(rng.random(n) < 0.8, 0xFFFFFFFF, 1 << rng.integers(0, 32, n)).astype(np.uint32)
    local = np.tile(IDENTITY, (n, 1))
    local[mesh - 2, 12:15] = boxes[:, :3]
    local[mesh - 1, 12:15] = boxes[:, 3:]
    aabb = np.tile(UNIT_BOX, (n, 1))
    aabb[mesh] = np.concatenate([boxes[:, :3], boxes[:, :3]], 1)
    og = ob.Graph.build(parent, flags, mask, local, aabb)
    ctx.set_topology(parent, flags, mask, aabb)
    ctx.set_local_matrices(local)
    for i in mesh.tolist():
        og.add_surface(i, [i - 2, i - 1])
        ctx.add_skinned_surface(i, [i - 2, i - 1], np.tile(IDENTITY, (2, 1)))
    og.L.orc_graph_drop_messages(og.h)
    og.update_hierarchical_data()
    ctx.update_and_cull([ef.ff for ef in frusta], fb.UPDATE_ALL, cam, pf)
    W = ctx.get_world_aabbs(mesh)
    want_box = np.where(boxes == 0, f32(0.0), boxes)  # a -0 bound folds as whichever zero came first; compare by value
    assert (W == want_box).all()
    census = {}
    check_visible(og, ctx, frusta, mesh, flags, mask, cam, pf, census)
    assert_census(census, frusta=frusta)


# ---- 5. lights: k_cull_lights ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_frusta", [1, 3, 8])
def test_light_lists_on_edge_points(ctx, n_frusta):
    """A light's world box is the unit box through its global transform; with a zero scale it is the point at its translation,
    exactly.  The lights sit on planes, on frustum corners, one ulp off them, and at huge / non-finite positions."""
    rng = np.random.default_rng(600 + n_frusta)
    frusta = pick_frusta(rng, n_frusta)
    pts = np.concatenate([ce.edge_points(ef, rng) for ef in frusta])
    pts = pts[rng.permutation(len(pts))]
    n = len(pts) + 1
    parent = np.zeros(n, np.uint32)
    parent[0] = NONE
    flags = np.full(n, fb.NODE_DEFAULT | fb.NODE_LIGHT, np.uint32)
    flags[0] = fb.NODE_DEFAULT
    local = np.tile(IDENTITY, (n, 1))
    local[1:, [0, 5, 10]] = 0.0
    local[1:, 12:15] = pts
    aabb = np.tile(UNIT_BOX, (n, 1))
    og = load(ctx, parent, flags, None, local, aabb)
    ctx.update_and_cull([ef.ff for ef in frusta], fb.UPDATE_ALL)
    ctx.cull_lights()
    nodes = np.arange(1, n, dtype=np.uint32)
    W = ctx.get_world_aabbs(nodes)
    assert bits_equal(W, og.world_bounding_boxes(nodes)).all()
    census = {}
    for f, ef in enumerate(frusta):
        got = ctx.get_visible_lights(f)
        assert np.array_equal(got, og.collect_lights(ef.fo)), ef.name  # same set, the reference's pool order
        assert np.array_equal(np.isin(nodes, got), ef.intersects(W)), ef.name
        for c, m in ce.classify(ef.planes, ef.corners, W).items():
            census[c] = census.get(c, 0) + int(m.sum())
    short = {c: census.get(c, 0) for c in ("point_plane", "point_corner", "pm_equal", "non_tame", "fallback_true") if census.get(c, 0) < 2}
    assert not short, (short, census)
    print("census", census)


# ---- 6. frusta built on the device: the shadow-map, observer and scene-shadow culls ---------------------------------------------
# Each runs in two phases: the first call gives the matrices the device builds its frusta from; edge boxes against those frusta
# (Frustum::from_view_projection_matrix of them) are added to the scene, and the call runs again.  Lights placed at edge points of
# the camera's or an observer's frustum (zero scale: the world box is the point, exactly) make shadow_light_gate decide on edges.
def append_nodes(sc, boxes=(), light_points=(), light_kind=fb.LIGHT_DIRECTIONAL):
    """Append to a ShadowScene renderable children of the root carrying `boxes` (identity local matrices) and shadow-casting
    lights at `light_points` (TRS records with zero scale).  Returns (box nodes, light nodes)."""
    from test_gpu_shadow_casters import local_from_trs

    nb, nl = len(boxes), len(light_points)
    k = nb + nl
    first = sc.n
    sc.n += k
    sc.parent = np.concatenate([sc.parent, np.zeros(k, np.uint32)])
    sc.flags = np.concatenate([sc.flags, np.full(nb, RENDER, np.uint32), np.full(nl, fb.NODE_DEFAULT | fb.NODE_LIGHT, np.uint32)])
    sc.mask = np.concatenate([sc.mask, np.full(k, 0xFFFFFFFF, np.uint32)])
    trs = np.zeros((k, 10), f32)
    trs[:, 6:10] = (1.0, 1.0, 1.0, 1.0)
    trs[nb:, 0:3] = np.asarray(light_points, f32).reshape(-1, 3)
    trs[nb:, 7:10] = 0.0
    local = np.tile(IDENTITY, (k, 1))
    if nl:
        local[nb:] = local_from_trs(trs[nb:])
    sc.local = np.concatenate([sc.local, local])
    sc.aabb = np.concatenate([sc.aabb, np.asarray(boxes, f32).reshape(-1, 6), np.tile(UNIT_BOX, (nl, 1))])
    sc.trs = np.concatenate([sc.trs, trs])
    lights = np.arange(first + nb, first + k, dtype=np.uint32)
    sc.lights = np.concatenate([sc.lights, lights])
    for x in lights.tolist():
        sc.sources[x] = (light_kind, f32(1.0), f32(10.0))
    return np.arange(first, first + nb, dtype=np.uint32), lights


def gate_points(ef, rng, n=40):
    """Edge points of a frustum for lights: finite and moderate (a light's maps are built around its position)."""
    pts = ce.edge_points(ef, rng)
    pts = pts[(np.abs(pts) < 1e6).all(1)]
    on_corner = (pts[:, None, :] == ef.corners[None]).all(2).any(1)  # every frustum corner, then a sample of the rest
    rest = pts[~on_corner]
    return np.concatenate([pts[on_corner], rest[rng.permutation(len(rest))[:max(0, n - int(on_corner.sum()))]]])


def map_key(m):
    return (int(m["light"]), int(m["face"]), int(m["cascade"]), m["view_projection"].tobytes())


def frusta_of_maps(maps, rng, k=4):
    """EdgeFrustum of up to k maps whose matrix has a frustum, keyed like map_key."""
    out = []
    for m in rng.permutation(len(maps)).tolist():
        if ob.frustum_from_vp(maps[m]["view_projection"]) is None:
            continue
        out.append((map_key(maps[m]), ce.EdgeFrustum.from_vp(f"map{m}", maps[m]["view_projection"])))
        if len(out) == k:
            break
    return out


def add_census(census, ef, boxes):
    for c, v in ce.classify(ef.planes, ef.corners, boxes).items():
        census[c] = census.get(c, 0) + int(v.sum())


@pytest.mark.parametrize("form", ["plain", "csm", "pruned"])
def test_shadow_maps_on_edge_boxes_of_their_own_frusta(ctx, form):
    """fyx_cull_shadow_casters, _csm and _pruned.  In the pruned form some edge boxes are static batches with edge-box children:
    the children are pruned from exactly the maps that render the batch.  In the csm and pruned forms directional lights sit at
    edge points of the camera frustum: a light gets cascades only where the camera's light list (its box) takes it."""
    from test_gpu_shadow_casters import ShadowScene, compare as compare_plain
    from test_gpu_shadow_csm import camera, compare as compare_csm, send_options
    from test_gpu_shadow_pruned import Pruners, pruned_cull
    from helpers import camera_frustum

    rng = np.random.default_rng(700 + ["plain", "csm", "pruned"].index(form))
    sc = ShadowScene(rng, 3000, 40, p_cast=0.9)
    pr = Pruners(sc) if form == "pruned" else None
    if pr:
        pr.add_random(rng)
    cam = camera()
    cam_fo = camera_frustum((0, 0, 0), (0, 0, -1), zfar=150.0)[0] if form == "plain" else cam[0]

    def load():
        og = sc.load(ctx)
        if pr:
            pr.send_ranges(ctx)
            og = pr.oracle()
        return og

    def run(og):
        if form == "plain":
            return compare_plain(ctx, og, sc)
        send_options(ctx, cam[2], {})
        if form == "csm":
            return compare_csm(ctx, og, sc, cam)
        return pruned_cull(ctx, og, sc, cam)[:2]

    maps, _ = run(load())
    picked = frusta_of_maps(maps, rng)
    assert len(picked) >= 2
    boxes = ce.all_boxes([ef for _, ef in picked], rng)
    gate = ce.EdgeFrustum("camera", *ob.frustum_planes_corners(cam_fo), fo=cam_fo)
    pts = gate_points(gate, rng) if form != "plain" else np.zeros((0, 3), f32)
    box_nodes, gate_lights = append_nodes(sc, boxes, pts)
    batch_of = {}
    if pr:
        for b in box_nodes[::12][:-1].tolist():  # a static batch with the next two edge boxes as its children
            sc.flags[b] |= np.uint32(fb.NODE_STATIC_BATCH)
            for c in (b + 1, b + 2):
                sc.parent[c] = b
                batch_of[c] = b
    maps2, entries = run(load())
    by_key = {map_key(m): m for m in maps2}
    W = ctx.get_world_aabbs(box_nodes)
    census, split = {}, 0
    for key, ef in picked:
        m = by_key[key]
        got = entries[m["first"]: m["first"] + m["count"]]
        want = ef.intersects(W)
        for c, b in batch_of.items():
            i, j = c - int(box_nodes[0]), b - int(box_nodes[0])
            split += int(want[i] and want[j])
            want[i] &= not want[j]
        assert np.array_equal(np.isin(box_nodes, got), want), (form, ef.name)
        add_census(census, ef, W)
    assert_census(census, frusta=[ef for _, ef in picked])
    if pr:
        assert split > 0  # some child is taken by the predicate and dropped because its batch is rendered
    if len(gate_lights):
        P = ctx.get_world_aabbs(gate_lights)
        lit = gate.intersects(P)
        with_maps = np.isin(gate_lights, maps2["light"])
        assert not (with_maps & ~lit).any()
        assert with_maps.any() and (~lit).any()
        gc = {}
        add_census(gc, gate, P)
        assert gc["point_plane"] > 0 and gc["point_corner"] > 0, gc


def test_scene_observers_on_edge_boxes_and_edge_lights(ctx):
    """fyx_cull_scene_observers: the observers' frusta are built on the device (to_dev_frustum); their visible lists and light
    lists (k_observer_lights) on edge boxes and edge-point lights of those frusta."""
    from test_gpu_observers import ObserverScene, key, observe

    rng = np.random.default_rng(800)
    s = ObserverScene(rng, 2000, 6, 2)
    og = s.load(ctx)
    table, _, _, _ = observe(ctx, og, s)
    picked = []
    for r in rng.permutation(len(table)).tolist():
        if ob.frustum_from_vp(table[r]["view_projection"]) is not None:
            picked.append((key([table[r]])[0], ce.EdgeFrustum.from_vp(f"observer{r}", table[r]["view_projection"])))
        if len(picked) == 4:
            break
    assert len(picked) >= 2
    boxes = ce.all_boxes([ef for _, ef in picked], rng)
    pts = np.concatenate([gate_points(ef, rng, 24) for _, ef in picked])
    box_nodes, light_nodes = append_nodes(s.sc, boxes, pts)
    og = s.load(ctx)
    table, entries, lights, _ = observe(ctx, og, s)
    rows = {key([r])[0]: r for r in table}
    W, P = ctx.get_world_aabbs(box_nodes), ctx.get_world_aabbs(light_nodes)
    census, lc = {}, {}
    for k, ef in picked:
        r = rows[k]
        got = entries[r["first"]: r["first"] + r["count"]]
        assert int(r["render_mask"]) != 0
        assert np.array_equal(np.isin(box_nodes, got), ef.intersects(W)), ef.name
        lg = lights[r["lights_first"]: r["lights_first"] + r["lights_count"]]
        assert np.array_equal(np.isin(light_nodes, lg), ef.intersects(P)), ef.name
        add_census(census, ef, W)
        add_census(lc, ef, P)
    assert_census(census, frusta=[ef for _, ef in picked])
    assert lc["point_plane"] > 0 and lc["point_corner"] > 0 and lc["fallback_true"] > 0, lc


def test_scene_shadow_maps_on_edge_boxes_and_edge_lights(ctx):
    """fyx_cull_scene_shadow_casters: edge boxes against the frusta of several of its maps, and directional lights at edge points
    of one observer's frustum — such a light is referenced by an observer only where that observer's light list takes it."""
    from test_gpu_scene_shadows import observe_and_shadow
    from test_gpu_observers import ObserverScene

    rng = np.random.default_rng(900)
    s = ObserverScene(rng, 2000, 6, 2)
    og = s.load(ctx)
    want, (maps, _, _) = observe_and_shadow(ctx, og, s)
    picked = frusta_of_maps(maps, rng)
    assert len(picked) >= 2
    obs = [o for o, w in enumerate(want) if ob.frustum_from_vp(w["view_projection"]) is not None]
    o_gate = obs[0]
    gate = ce.EdgeFrustum.from_vp("observer", want[o_gate]["view_projection"])
    boxes = ce.all_boxes([ef for _, ef in picked], rng)
    box_nodes, gate_lights = append_nodes(s.sc, boxes, gate_points(gate, rng))
    og = s.load(ctx)
    want, (maps2, entries, refs) = observe_and_shadow(ctx, og, s)
    W = ctx.get_world_aabbs(box_nodes)
    census = {}
    rows = [map_key(m) for m in maps2]
    for k, ef in picked:
        hits = [i for i, rk in enumerate(rows) if rk == k]
        assert hits, ef.name
        for i in hits:
            m = maps2[i]
            got = entries[m["first"]: m["first"] + m["count"]]
            assert np.array_equal(np.isin(box_nodes, got), ef.intersects(W)), ef.name
        add_census(census, ef, W)
    assert_census(census, frusta=[ef for _, ef in picked])
    # the gate: an observer references a gate light's maps only if its own frustum takes the light's point
    P = ctx.get_world_aabbs(gate_lights)
    fr = {o: ce.EdgeFrustum.from_vp(f"o{o}", w["view_projection"]) for o, w in enumerate(want)
          if ob.frustum_from_vp(w["view_projection"]) is not None}
    seen = np.zeros(len(gate_lights), bool)
    for r in refs:
        light = int(maps2[int(r["map"])]["light"])
        if light in gate_lights:
            i = int(np.flatnonzero(gate_lights == light)[0])
            o = int(r["observer"])
            assert o in fr and fr[o].intersects(P[i:i + 1])[0], (o, light)
            seen[i] |= o == o_gate
    lit = gate.intersects(P)
    assert seen.any() and (~lit).any() and not (seen & ~lit).any()
