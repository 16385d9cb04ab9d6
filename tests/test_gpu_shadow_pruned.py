"""Shadow maps with each map's own LOD filter and static-batch pruning: fyx_cull_shadow_casters_pruned against the oracle.

The reference builds one RenderDataBundleStorage::from_graph per shadow map (renderer/bundle.rs:873-1009), with that map's
observer: the light's position, z_near 0.01 and z_far light_radius for spot maps and cube faces, the look_at_lh eye
center + light_direction and the slice's depths for cascade i (shadow/csm.rs:195-270).  So map m's list is
og.from_graph_lod(map frustum, observer translation, z_near, z_far, camera mask, shadow pass).  The map table itself must
be the one fyx_cull_shadow_casters_csm gives, view_projection bit for bit."""
import numpy as np
import pytest

import csm_oracle as co
import fyrox_b200 as fb
import oracle_binding as ob
import shadow_oracle as so
from fyrox_b200 import _lib as L
from test_gpu_shadow_casters import ShadowScene, in_view, local_from_trs, rand_quat
from test_gpu_shadow_csm import camera, same_bits, send_options

pytestmark = pytest.mark.gpu

f32 = np.float32
SETTINGS = (40.0, 40.0, 1, 1)
DIR = fb.LIGHT_DIRECTIONAL
LEVELS = [(0.0, 0.4), (0.4, 1.2), (1.2, 6.0)]


class Pruners:
    """LOD objects (one range per node, last write wins as fyx_set_lod_ranges resolves it) and static batches of a
    ShadowScene, on both sides.  The oracle is rebuilt from the scene's columns after every change."""

    def __init__(self, sc):
        self.sc = sc
        self.ranges = {}

    def add_random(self, rng, p_lod=0.03, p_batch=0.02):
        sc = self.sc
        has_child = np.zeros(sc.n, bool)
        has_child[sc.parent[1:]] = True
        cand = np.flatnonzero(np.arange(sc.n) > 0)
        for x in rng.choice(cand, max(1, int(p_lod * sc.n)), replace=False).tolist():
            self.ranges[int(x)] = LEVELS[int(rng.integers(0, len(LEVELS)))]
        parents = np.flatnonzero(has_child & ((sc.flags & fb.NODE_RENDERABLE) != 0))
        parents = parents[parents > 0]
        batches = rng.choice(parents, max(1, int(p_batch * sc.n)), replace=False)
        sc.flags[batches] |= np.uint32(fb.NODE_STATIC_BATCH)
        return batches

    def send_ranges(self, ctx, nodes=None):
        nodes = sorted(self.ranges) if nodes is None else nodes
        if nodes:
            be = np.array([self.ranges.get(int(x), (np.nan, np.nan)) for x in nodes], f32)
            ctx.set_lod_ranges(be, np.array(nodes, np.uint32))

    def oracle(self):
        sc = self.sc
        og = ob.Graph.build(sc.parent, sc.flags, sc.mask, sc.local, sc.aabb)
        if self.ranges:
            xs = sorted(self.ranges)
            og.set_lod_group(0, [(self.ranges[x][0], self.ranges[x][1], [x]) for x in xs])
        og.update_hierarchical_data()
        return og


def observers(og, sc, maps, oc):
    """(translation, z_near, z_far) of every map of the table."""
    out = []
    for m in maps:
        light = int(m["light"])
        g = og.global_transform(light)
        if sc.sources[light][0] == DIR:
            with np.errstate(all="ignore"):
                zn, zf = co.cascade_depths(oc, oc.options.get(light, co.CSM_DEFAULT), int(m["cascade"]))
                light_direction = -so.try_normalize(g[4:7].astype(f32), so.F32_EPSILON, (0.0, 1.0, 0.0))
                center = co.frustum_center(co.slice_corners(oc, zn, zf))
                out.append((center + light_direction, f32(zn), f32(zf)))
        else:
            scl = np.asarray(sc.scale().get(light, (1.0, 1.0, 1.0)), f32)
            radius = f32(np.fmax(np.fmax(scl[0], scl[1]), scl[2])) * f32(sc.sources[light][2])
            out.append((g[12:15].astype(f32), f32(0.01), radius))
    return out


def pruned_cull(ctx, og, sc, cam, eye=(0.0, 0.0, 0.0), cam_mask=0xFFFFFFFF, settings=SETTINGS, csm=True):
    """The pruned cull against the oracle: the table equals the unpruned oracle's (and thus _csm's), every list
    from_graph_lod with the map's observer.  Returns (maps, entries, oracle lists, observers)."""
    fo, ff, oc, fc = cam
    ctx.cull([ff], cam_mask=[cam_mask])
    ctx.cull_shadow_casters(0, np.array(eye, f32), *settings, csm_camera=fc if csm else None, prune=True)
    maps, entries = ctx.get_shadow_maps()
    want = co.shadow_maps(og, sc.flags, fo, eye, cam_mask, settings, sc.sources, sc.scale(), csm=oc if csm else None)
    assert [(int(m["light"]), int(m["face"]), int(m["cascade"])) for m in maps] == [(w[0], w[1], w[2]) for w in want]
    obs = observers(og, sc, maps, oc)
    lists = []
    for m, w, (t, zn, zf) in zip(maps, want, obs):
        assert same_bits(m["view_projection"], w[3])
        fr = ob.frustum_from_vp(w[3]) or so.default_frustum()
        vis = np.sort(og.from_graph_lod(fr, t, zn, zf, cam_mask, shadow_pass=True))
        got = np.sort(entries[m["first"]: m["first"] + m["count"]])
        assert np.array_equal(got, vis), (int(m["light"]), int(m["face"]), int(m["cascade"]), len(got), len(vis))
        lists.append(vis)
    return maps, entries, lists, obs


def unpruned_table(sc, cam, eye=(0.0, 0.0, 0.0), settings=SETTINGS, csm=True):
    """_csm on the same scene without its ranges and batch flags, on a context of its own: the table and the lists."""
    fo, ff, oc, fc = cam
    flags = sc.flags
    sc.flags = flags & ~np.uint32(fb.NODE_STATIC_BATCH)
    try:
        with fb.Context() as c2:
            sc.load(c2)
            c2.cull([ff])
            c2.cull_shadow_casters(0, np.array(eye, f32), *settings, csm_camera=fc if csm else None)
            return c2.get_shadow_maps()
    finally:
        sc.flags = flags


def table_key(maps):
    return [(int(m["light"]), int(m["face"]), int(m["cascade"]), m["view_projection"].tobytes()) for m in maps]


def non_vacuous(og, sc, lists, obs, pr):
    """A LOD object hidden in one map and visible in another; a static batch that prunes its children in one map and
    lets them be visited in another."""
    lod_split = False
    if pr.ranges:
        xs = np.array(sorted(pr.ranges))
        filt = np.stack([og.lod_filter(t, zn, zf)[xs] for t, zn, zf in obs]) if obs else np.zeros((0, xs.size))
        lod_split = bool(np.any(filt.any(axis=0) & ~filt.all(axis=0)))
    children = {}
    for i in range(1, sc.n):
        children.setdefault(int(sc.parent[i]), []).append(i)
    batch_split = False
    batches = np.flatnonzero((sc.flags & fb.NODE_STATIC_BATCH) != 0).tolist()
    sets = [set(v.tolist()) for v in lists]
    for b in batches:
        ch = children.get(b, [])
        rendered = [b in s for s in sets]
        if any(rendered) and any(not r and any(c in s for c in ch) for r, s in zip(rendered, sets)):
            batch_split = True
            break
    return lod_split, batch_split


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_random_scenes_match_the_oracle(ctx, seed):
    rng = np.random.default_rng(2100 + seed)
    sc = ShadowScene(rng, 4000, 30, p_cast=0.9)
    pr = Pruners(sc)
    pr.add_random(rng)
    og = sc.load(ctx)
    pr.send_ranges(ctx)
    og = pr.oracle()
    cam = camera()
    send_options(ctx, cam[2], {})
    maps, entries, lists, obs = pruned_cull(ctx, og, sc, cam)
    assert len(maps) > 6 and any(sc.sources[int(m["light"])][0] == DIR for m in maps)
    assert non_vacuous(og, sc, lists, obs, pr) == (True, True)
    # the same table as _csm gives on the scene without ranges and batches
    m0, _ = unpruned_table(sc, cam)
    assert table_key(m0) == table_key(maps)
    # the old calls refuse this scene (ranges with observers; static batches)
    ctx.cull([cam[1]])
    with pytest.raises(fb.FyxError) as e:
        ctx.cull_shadow_casters(0, np.zeros(3, f32), *SETTINGS, csm_camera=cam[3])
    assert e.value.code == L.FYX_ERR_STATE
    # no cascades (NULL camera), another camera position and mask
    pruned_cull(ctx, og, sc, cam, csm=False)
    cam2 = camera(eye=(3.0, 1.0, -10.0), target=(2.0, 0.5, -11.0), z_near=0.5, z_far=90.0)
    cam2[2].options = {}
    pruned_cull(ctx, og, sc, cam2, eye=(3.0, 1.0, -10.0), cam_mask=0x1, settings=(25.0, 60.0, 1, 1))


def chain_scene(rng):
    """The random base of test_both_rules_at_once, which adds chains with nested LOD objects, a batch under a LOD object, a
    node that is both, a batch without cast_shadows, a batch with frustum_culling off and a batch with a tiny box."""
    sc = ShadowScene(rng, 1500, 10, kinds=(1, 2), p_cast=1.0)
    in_view(rng, sc)
    return sc


def test_both_rules_at_once(ctx):
    rng = np.random.default_rng(2200)
    sc = chain_scene(rng)
    n0 = 1300
    # chains n0 -> n0+1 -> ... hang below the root near the lights: positions relative to the parent are small
    chain = list(range(n0, n0 + 40))
    for k, i in enumerate(chain):
        sc.parent[i] = 0 if k % 8 == 0 else i - 1
        sc.trs[i, 0:3] = sc.trs[int(sc.lights[k % len(sc.lights)]), 0:3] + rng.uniform(-1.5, 1.5, 3) if k % 8 == 0 else rng.uniform(-0.3, 0.3, 3)
        sc.trs[i, 3:7] = (0, 0, 0, 1)
        sc.flags[i] = fb.NODE_DEFAULT | fb.NODE_RENDERABLE
    sc.local[chain] = local_from_trs(sc.trs[chain])
    pr = Pruners(sc)
    blocks = [chain[b: b + 8] for b in range(0, 40, 8)]
    # block 0: nested LOD objects (outer and inner ranges differ)
    pr.ranges[blocks[0][1]] = (0.0, 0.5)
    pr.ranges[blocks[0][3]] = (0.3, 6.0)
    # block 1: a static batch under a LOD object, and a node that is both
    pr.ranges[blocks[1][1]] = (0.2, 6.0)
    sc.flags[blocks[1][2]] |= np.uint32(fb.NODE_STATIC_BATCH)
    pr.ranges[blocks[1][4]] = (0.0, 0.6)
    sc.flags[blocks[1][4]] |= np.uint32(fb.NODE_STATIC_BATCH)
    # block 2: a static batch without cast_shadows (never rendered in a shadow map: children visited)
    sc.flags[blocks[2][1]] |= np.uint32(fb.NODE_STATIC_BATCH)
    sc.flags[blocks[2][1]] &= ~np.uint32(fb.NODE_CAST_SHADOWS)
    # block 3: a static batch with frustum_culling off (rendered in every map that passes the mask)
    sc.flags[blocks[3][1]] |= np.uint32(fb.NODE_STATIC_BATCH)
    sc.flags[blocks[3][1]] &= ~np.uint32(fb.NODE_FRUSTUM_CULLING)
    # block 4: a static batch with a tiny box (outside many maps: its children are visited there)
    sc.flags[blocks[4][1]] |= np.uint32(fb.NODE_STATIC_BATCH)
    sc.trs[blocks[4][1], 0:3] = (0.0, 0.0, 0.05)
    sc.local[blocks[4][1]] = local_from_trs(sc.trs[blocks[4][1]: blocks[4][1] + 1])[0]
    sc.aabb[blocks[4][1]] = (-0.01, -0.01, -0.01, 0.01, 0.01, 0.01)
    og = sc.load(ctx)
    pr.send_ranges(ctx)
    og = pr.oracle()
    cam = camera()
    send_options(ctx, cam[2], {})
    maps, entries, lists, obs = pruned_cull(ctx, og, sc, cam, settings=(200.0, 200.0, 1, 1))
    assert len(maps) >= 10
    sets = [set(v.tolist()) for v in lists]
    # the batch without cast_shadows is never listed, its child is listed somewhere
    assert not any(blocks[2][1] in s for s in sets) and any(blocks[2][2] in s for s in sets)


def test_more_than_64_maps(ctx):
    """40 point lights: ~240 maps, W > 2 words per pruner row, word boundaries crossed."""
    rng = np.random.default_rng(2300)
    sc = ShadowScene(rng, 6000, 40, spread=15.0, depth_z=(-40.0, -3.0), kinds=(2,), p_cast=1.0)
    in_view(rng, sc)
    pr = Pruners(sc)
    pr.add_random(rng, p_lod=0.05, p_batch=0.03)
    og = sc.load(ctx)
    pr.send_ranges(ctx)
    og = pr.oracle()
    cam = camera()
    maps, entries, lists, obs = pruned_cull(ctx, og, sc, cam, settings=(500.0, 500.0, 1, 1), csm=False)
    assert len(maps) > 200
    assert non_vacuous(og, sc, lists, obs, pr) == (True, True)
    m0, _ = unpruned_table(sc, cam, settings=(500.0, 500.0, 1, 1), csm=False)
    assert table_key(m0) == table_key(maps)


def test_degenerate_depth_ranges(ctx):
    """A point light with light_radius == 0.01 (z_far == z_near: the normalised distance is ±inf or NaN) and a cascade
    whose slice collapses to Frustum::default."""
    rng = np.random.default_rng(2400)
    sc = ShadowScene(rng, 2500, 12, kinds=(DIR, 2), p_cast=1.0)
    in_view(rng, sc)
    point = [n for n in sc.lights.tolist() if sc.sources[n][0] == fb.LIGHT_POINT][0]
    sc.sources[point] = (fb.LIGHT_POINT, f32(0.0), f32(0.01))
    sc.trs[point, 7:10] = 1.0
    sc.local[point] = local_from_trs(sc.trs[point: point + 1])[0]
    pr = Pruners(sc)
    pr.add_random(rng, p_lod=0.05)
    pr.ranges[int(rng.integers(1, sc.n))] = (-np.inf, np.inf)
    og = sc.load(ctx)
    pr.send_ranges(ctx)
    og = pr.oracle()
    for kw in (dict(), dict(frame=(640.0, 0.0))):
        cam = camera(**kw)
        dirs = [n for n in sc.lights.tolist() if sc.sources[n][0] == DIR]
        send_options(ctx, cam[2], {dirs[0]: (0, (0.1, 0.1, 30.0))})
        pruned_cull(ctx, og, sc, cam, settings=(500.0, 500.0, 1, 1))


def test_state_changes_between_calls(ctx):
    rng = np.random.default_rng(2500)
    sc = ShadowScene(rng, 3000, 16, kinds=(1, 2, 3), p_cast=0.95)
    pr = Pruners(sc)
    batches = pr.add_random(rng)
    og = sc.load(ctx)
    pr.send_ranges(ctx)
    cam = camera()
    send_options(ctx, cam[2], {})
    pruned_cull(ctx, pr.oracle(), sc, cam)
    # a range removed with begin = NaN, then added again
    x = sorted(pr.ranges)[0]
    r = pr.ranges.pop(x)
    ctx.set_lod_ranges(np.array([[np.nan, np.nan]], f32), np.array([x], np.uint32))
    pruned_cull(ctx, pr.oracle(), sc, cam)
    pr.ranges[x] = r
    pr.send_ranges(ctx, [x])
    pruned_cull(ctx, pr.oracle(), sc, cam)
    # FYX_NODE_STATIC_BATCH set on new nodes, then cleared on old ones, through fyx_set_flags
    extra = rng.choice(np.flatnonzero(sc.flags & fb.NODE_RENDERABLE), 40, replace=False)
    sc.flags[extra] |= np.uint32(fb.NODE_STATIC_BATCH)
    ctx.set_flags(sc.flags[extra], extra.astype(np.uint32))
    ctx.update_transforms(fb.UPDATE_ALL)
    pruned_cull(ctx, pr.oracle(), sc, cam)
    sc.flags[batches] &= ~np.uint32(fb.NODE_STATIC_BATCH)
    ctx.set_flags(sc.flags[batches], batches.astype(np.uint32))
    ctx.update_transforms(fb.UPDATE_ALL)
    pruned_cull(ctx, pr.oracle(), sc, cam)
    # fyx_set_topology re-parents a static batch and a LOD object (the ranges stay with their node indices); a parent
    # always has a smaller index than its child here, so the graph stays a forest
    b = int(extra[extra > 2][0])
    lod = [x for x in sorted(pr.ranges) if x > 2][0]
    for node in (b, lod):
        sc.parent[node] = int(rng.integers(0, node - 1)) if sc.parent[node] == node - 1 else node - 1
    ctx.set_topology(sc.parent, sc.flags, sc.mask, sc.aabb)
    ctx.set_local_matrices(sc.local)
    ctx.set_local_trs(sc.trs[sc.lights], sc.lights)
    ctx.update_transforms(fb.UPDATE_ALL)
    pruned_cull(ctx, pr.oracle(), sc, cam)
    # lights moved by TRS
    moved = sc.lights[::2]
    sc.trs[moved, 0:3] += rng.uniform(-4.0, 4.0, (len(moved), 3)).astype(f32)
    sc.trs[moved, 3:7] = rand_quat(rng, len(moved))
    sc.local[moved] = local_from_trs(sc.trs[moved])
    ctx.set_local_trs(sc.trs[moved], moved)
    ctx.update_transforms(fb.UPDATE_INCREMENTAL)
    pruned_cull(ctx, pr.oracle(), sc, cam)


def test_without_pruners_equals_csm(ctx):
    rng = np.random.default_rng(2600)
    sc = ShadowScene(rng, 4000, 24)
    og = sc.load(ctx)
    cam = camera()
    send_options(ctx, cam[2], {})
    fo, ff, oc, fc = cam
    ctx.cull([ff])
    n0 = ctx.kernel_launch_count()
    ctx.cull_shadow_casters(0, np.zeros(3, f32), *SETTINGS, csm_camera=fc)
    n1 = ctx.kernel_launch_count()
    m0, e0 = ctx.get_shadow_maps()
    ctx.cull_shadow_casters(0, np.zeros(3, f32), *SETTINGS, csm_camera=fc, prune=True)
    n2 = ctx.kernel_launch_count()
    m1, e1 = ctx.get_shadow_maps()
    assert n2 - n1 == n1 - n0
    assert m0.tobytes() == m1.tobytes()
    for m in m1:
        sl = slice(int(m["first"]), int(m["first"] + m["count"]))
        assert np.array_equal(np.sort(e0[sl]), np.sort(e1[sl]))
    pruned_cull(ctx, og, sc, cam)
    # ranges that were all removed again count as none
    ctx.set_lod_ranges(np.array([[0.0, 0.1]], f32), np.array([5], np.uint32))
    ctx.set_lod_ranges(np.array([[np.nan, np.nan]], f32), np.array([5], np.uint32))
    ctx.cull([ff])
    n3 = ctx.kernel_launch_count()
    ctx.cull_shadow_casters(0, np.zeros(3, f32), *SETTINGS, csm_camera=fc, prune=True)
    assert ctx.kernel_launch_count() - n3 == n1 - n0


def test_pack_after_a_pruned_cull(ctx):
    """The pruned lists feed fyx_pack_shadow_instances unchanged: each instance as the oracle's orc_node_instance; a static
    batch carries the identity world matrix, so world · VP == VP."""
    rng = np.random.default_rng(2700)
    sc = ShadowScene(rng, 3000, 10, spread=12.0, depth_z=(-30.0, -2.0), kinds=(1, 2, 3), p_cast=1.0)
    in_view(rng, sc)
    pr = Pruners(sc)
    pr.add_random(rng, p_lod=0.04, p_batch=0.04)
    og = sc.load(ctx)
    pr.send_ranges(ctx)
    og = pr.oracle()
    ctx.enable_instances()
    cam = camera()
    send_options(ctx, cam[2], {})
    maps, entries, lists, obs = pruned_cull(ctx, og, sc, cam, settings=(200.0, 200.0, 1, 1))
    ctx.pack_shadow_instances()
    ctx.pack_shadow_bone_matrices()
    views = {}
    n_batch = n_inst = 0
    for k, m in enumerate(maps):
        light = int(m["light"])
        if sc.sources[light][0] == DIR:
            if light not in views:
                views[light] = co.cascade_views(og, light, cam[2])
            view = views[light][int(m["cascade"])]
        else:
            g = og.global_transform(light)
            position = g[12:15].astype(f32)
            if sc.sources[light][0] == so.LIGHT_SPOT:
                emit = so.try_normalize(g[4:7].astype(f32), so.F32_EPSILON, (0.0, 0.0, 1.0))
                up = so.try_normalize(g[8:11].astype(f32), so.F32_EPSILON, (0.0, 1.0, 0.0))
                view = ob.look_at_rh(position, position - emit, up)
            else:
                look, up = so.CUBE_FACES[int(m["face"])]
                view = ob.look_at_rh(position, position + np.array(look, f32), np.array(up, f32))
        inst = ctx.get_shadow_instances(k)
        assert np.array_equal(np.sort(inst["node"]), lists[k])
        vp = m["view_projection"].copy()
        for i in range(inst["node"].size):
            nd = int(inst["node"][i])
            si, ww, wvp = og.instance(nd, view, vp)
            assert int(inst["sort_index"][i]) == si
            assert inst["world"][i].tobytes() == ww.tobytes() and inst["wvp"][i].tobytes() == wvp.tobytes()
            if sc.flags[nd] & fb.NODE_STATIC_BATCH:
                assert inst["world"][i].tobytes() == np.eye(4, dtype=f32).tobytes()
                assert np.array_equal(inst["wvp"][i].reshape(16), vp)
                n_batch += 1
            assert ctx.get_shadow_bone_matrix_block(k, i) is None
            n_inst += 1
    assert n_batch > 0 and n_inst > 100


def test_errors_match_csm(ctx):
    rng = np.random.default_rng(2800)
    sc = ShadowScene(rng, 500, 6)
    pr = Pruners(sc)
    pr.add_random(rng)
    sc.load(ctx)
    pr.send_ranges(ctx)
    t = np.zeros(3, f32)
    fo, ff, oc, fc = camera()

    def code_of(fn):
        with pytest.raises(fb.FyxError) as e:
            fn()
        return e.value.code

    run = lambda f=0, cam=fc: ctx.cull_shadow_casters(f, t, csm_camera=cam, prune=True)  # noqa: E731
    assert code_of(run) == L.FYX_ERR_STATE  # no cull yet
    ctx.cull([ff])
    assert code_of(lambda: run(1)) == L.FYX_ERR_INVALID_ARGUMENT
    bad = camera()[3]
    bad.projection = 7
    assert code_of(lambda: run(0, bad)) == L.FYX_ERR_INVALID_ARGUMENT
    run()
    ctx.render_prep(frusta=[ff], async_=True, readback_visible=True, do_palettes=False, do_skin=False)
    assert code_of(run) == L.FYX_ERR_STATE  # a frame in flight
    ctx.frame_wait()
    run()
    run(0, None)
    # the unpruned calls still refuse this scene
    assert code_of(lambda: ctx.cull_shadow_casters(0, t, csm_camera=fc)) == L.FYX_ERR_STATE
    assert code_of(lambda: ctx.cull_shadow_casters(0, t)) == L.FYX_ERR_STATE


def test_one_million_nodes_compared_in_full(ctx):
    rng = np.random.default_rng(2900)
    sc = ShadowScene(rng, 1_000_000, 10, spread=40.0, rotate_all=False, kinds=(2,), p_cast=1.0)
    in_view(rng, sc)
    for k, node in enumerate(sc.lights.tolist()):
        sc.sources[node] = (DIR, f32(0.0), f32(0.0)) if k < 2 else (fb.LIGHT_POINT, f32(0.0), f32(rng.uniform(4.0, 12.0)))
    pr = Pruners(sc)
    pr.add_random(rng, p_lod=0.01, p_batch=0.001)
    og = sc.load(ctx)
    pr.send_ranges(ctx)
    og = pr.oracle()
    cam = camera()
    send_options(ctx, cam[2], {})
    maps, entries, lists, obs = pruned_cull(ctx, og, sc, cam, settings=(200.0, 200.0, 1, 1))
    assert len(maps) >= 30 and len(entries) > 100_000
