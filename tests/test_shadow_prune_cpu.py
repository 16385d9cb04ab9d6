"""The pruned shadow cull (fyx_cull_shadow_casters_pruned) does not walk the graph per map as the reference does
(renderer/bundle.rs:988-1004): it keeps one u32 per slot (the nearest pruner on the node's path, a pruner being a LOD object
or a static batch), two rows of ceil(maps / 32) words per pruner, filled parents first,

    self_hidden[p]     = children_hidden[anc(p)] | lod_out(p, m)
    children_hidden[p] = self_hidden[p] | (static_batch(p) && rendered(p, m))

and masks each node's own test with one bit of the right row.  This file restates that scheme in numpy (pruner ids in slot
order, one pass per hierarchy level, bits packed in u32 words) and checks it against the oracle's pruned DFS,
orc_from_graph_lod, on small random forests with 1, 33 and 70 maps, so that rows of one, two and three words are crossed."""
import numpy as np
import pytest

import fyrox_b200 as fb
import oracle_binding as ob

f32 = np.float32
NONE = 0xFFFFFFFF
SELF = 1 << 31


def random_forest(rng, n):
    """Parents always before their children; a few orphans outside the root's tree; translation-only locals."""
    parent = np.zeros(n, np.uint32)
    parent[0] = NONE
    parent[1:] = (rng.random(n - 1) * np.arange(1, n)).astype(np.uint32)
    orphan = rng.random(n) < 0.02
    orphan[0] = False
    parent[orphan] = NONE
    flags = np.full(n, fb.NODE_DEFAULT | fb.NODE_RENDERABLE, np.uint32)
    flags[rng.random(n) < 0.05] &= ~np.uint32(fb.NODE_CAST_SHADOWS)
    flags[rng.random(n) < 0.05] &= ~np.uint32(fb.NODE_FRUSTUM_CULLING)
    flags[0] = fb.NODE_DEFAULT
    mask = np.where(rng.random(n) < 0.9, 0xFFFFFFFF, 2).astype(np.uint32)
    local = np.tile(np.eye(4, dtype=f32).reshape(16), (n, 1))
    local[1:, 12:15] = rng.uniform(-6.0, 6.0, (n - 1, 3))
    h = rng.uniform(0.2, 1.5, (n, 3)).astype(f32)
    aabb = np.concatenate([-h, h], axis=1)
    return parent, flags, mask, local, aabb


def random_maps(rng, k):
    """k maps: (frustum, observer translation, z_near, z_far), some with a zero or negative depth range."""
    out = []
    for i in range(k):
        eye = rng.uniform(-12.0, 12.0, 3).astype(f32)
        target = rng.uniform(-4.0, 4.0, 3).astype(f32)
        zn = f32(0.01)
        zf = f32(rng.uniform(3.0, 30.0)) if i % 11 else f32(0.01) if i % 2 else f32(-2.0)
        fr = ob.frustum_from_vp(ob.mat4_mul(ob.perspective(1.0, float(rng.uniform(0.5, 2.0)), 0.1, 40.0), ob.look_at_rh(eye, target, (0.0, 1.0, 0.0))))
        out.append((fr, eye, zn, zf))
    return out


def pack(bits):
    """bool per map -> u32 words, map m at bit m % 32 of word m // 32"""
    w = np.zeros((len(bits) + 31) // 32, np.uint32)
    for m in np.flatnonzero(bits):
        w[m >> 5] |= np.uint32(1 << (m & 31))
    return w


def emulate(parent, is_lod, is_batch, raw, lod_out):
    """The device scheme.  raw[m, i]: node i is in map m's list without any pruning (its own test); lod_out[m, i]: node i's
    LOD range rejects map m's observer.  Returns the lists."""
    n_maps, n = raw.shape
    words = (n_maps + 31) // 32
    depth = np.zeros(n, np.int64)
    for i in range(n):  # parents come first
        depth[i] = 0 if parent[i] == NONE else depth[parent[i]] + 1
    order = np.lexsort((np.arange(n), depth))  # slot order: (depth, node index)
    pruner = is_lod | is_batch
    pid = {}
    for i in order:
        if pruner[i]:
            pid[int(i)] = len(pid)
    # the column: mark the pruners, then one pass per level, parents first
    col = np.full(n, NONE, np.uint64)
    anc = np.full(len(pid), NONE, np.uint64)
    for i, p in pid.items():
        col[i] = p | SELF
    for i in order:
        pv = col[parent[i]] if parent[i] != NONE else NONE
        up = NONE if pv == NONE else int(pv) & ~SELF
        if col[i] != NONE:
            anc[int(col[i]) & ~SELF] = up
        else:
            col[i] = up
    # the table, pruners in id order (ancestors have smaller ids)
    rows = np.zeros((len(pid), 2, words), np.uint32)
    for i, p in pid.items():
        a = int(anc[p])
        own = rows[a, 1].copy() if a != NONE else np.zeros(words, np.uint32)
        if is_lod[i]:
            own |= pack(lod_out[:, i])
        rows[p, 0] = own
        rows[p, 1] = own | (pack(raw[:, i]) if is_batch[i] else 0)
    lists = [[] for _ in range(n_maps)]
    for i in range(n):
        c = int(col[i])
        row = np.zeros(words, np.uint32) if c == NONE else rows[c & ~SELF, 0 if c & SELF else 1]
        for m in np.flatnonzero(raw[:, i]):
            if not (int(row[m >> 5]) >> (m & 31)) & 1:
                lists[m].append(i)
    return [np.array(sorted(x), np.uint32) for x in lists]


@pytest.mark.parametrize("n_maps", [1, 33, 70])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_column_and_table_match_the_pruned_dfs(n_maps, seed):
    rng = np.random.default_rng(3100 + 7 * seed + n_maps)
    n = 400
    parent, flags, mask, local, aabb = random_forest(rng, n)
    is_batch = (rng.random(n) < 0.08) & (np.arange(n) > 0)
    lod_nodes = rng.choice(np.arange(1, n), 30, replace=False)
    is_lod = np.zeros(n, bool)
    is_lod[lod_nodes] = True
    is_batch[lod_nodes[:5]] = True  # nodes that are both
    ranges = {int(x): [(0.0, 0.4), (0.3, 1.0), (0.8, 5.0)][k % 3] for k, x in enumerate(lod_nodes.tolist())}
    maps = random_maps(rng, n_maps)
    cam_mask = 0xFFFFFFFF if seed != 2 else 1
    # the raw tests: a graph without batches and ranges
    plain = ob.Graph.build(parent, flags, mask, local, aabb)
    plain.update_hierarchical_data()
    raw = np.zeros((n_maps, n), bool)
    for m, (fr, _, _, _) in enumerate(maps):
        raw[m, plain.from_graph(fr, cam_mask, shadow_pass=True)] = True
    # the full graph
    full_flags = flags | np.where(is_batch, fb.NODE_STATIC_BATCH, 0).astype(np.uint32)
    og = ob.Graph.build(parent, full_flags, mask, local, aabb)
    og.set_lod_group(0, [(ranges[x][0], ranges[x][1], [x]) for x in sorted(ranges)])
    og.update_hierarchical_data()
    lod_out = np.zeros((n_maps, n), bool)
    with np.errstate(all="ignore"):
        for m, (_, t, zn, zf) in enumerate(maps):
            lod_out[m] = ~og.lod_filter(t, zn, zf)
    got = emulate(parent, is_lod, is_batch, raw, lod_out)
    pruned_any = False
    for m, (fr, t, zn, zf) in enumerate(maps):
        want = np.sort(og.from_graph_lod(fr, t, zn, zf, cam_mask, shadow_pass=True)).astype(np.uint32)
        assert np.array_equal(got[m], want), (m, got[m].size, want.size)
        pruned_any |= want.size < int(raw[m].sum())
    assert pruned_any
