"""Context lifetime: every allocating path of one context, then fyx_destroy, several times in one process; and the multi-GPU
exchange set up, used, torn down by a second fyx_comm_init and used again on a single rank.

Later rounds must reproduce the first round bit for bit: state freed by one context (device and pinned buffers, events,
streams) must not leak into the next, and a context must not depend on what an earlier one left behind."""
import numpy as np
import pytest

import fyrox_b200 as fb
import oracle_binding as ob
from fyrox_b200 import _lib as L
from fyrox_b200.scenegen import Scene
from helpers import NONE, cube_frusta

pytestmark = pytest.mark.gpu

f32 = np.float32
N_NODES, N_UNITS, VERTS = 20000, 8, 700


def _position_animation(nodes, rng):
    """One animation: a linear position track of 3 curves per node."""
    tracks = np.zeros(len(nodes), fb.Context.TRACK_DTYPE)
    keys = []
    for k, node in enumerate(nodes):
        tracks[k]["target_node"], tracks[k]["binding"], tracks[k]["value_kind"] = node, L.BIND_POSITION, L.TV_VECTOR3
        tracks[k]["enabled"], tracks[k]["n_curves"] = 1, 3
        for c in range(3):
            tracks[k]["first_key"][c], tracks[k]["n_keys"][c] = len(keys), 2
            keys.append((0.0, float(rng.uniform(-20, 20)), L.KEY_LINEAR, 0.0, 0.0))
            keys.append((1.0, float(rng.uniform(-20, 20)), L.KEY_LINEAR, 0.0, 0.0))
    return tracks, np.array(keys, fb.Context.KEY_DTYPE)


def _every_feature_round():
    """One context through every allocating path; returns its outputs by name."""
    rng = np.random.default_rng(2024)
    sc = Scene(N_NODES, n_units=N_UNITS, verts_per_unit=VERTS)
    n = sc.capacity
    units = set()
    for u in range(sc.n_units):
        units.add(sc.unit_mesh_node(u))
        units.update(int(b) for b in sc.unit_bone_nodes(u))
    free = np.array([i for i in range(1, n) if i not in units and sc.parent[i] != NONE], np.uint32)
    pick = rng.permutation(free)
    lights, probes, lod, statics_nodes, late = pick[:24], pick[24:32], pick[32:72], pick[72:122], pick[122:322]
    flags = sc.flags.copy()
    flags[lights] |= fb.NODE_LIGHT
    flags[probes] |= fb.NODE_REFLECTION_PROBE
    aabb = sc.local_aabb.copy()
    _, ffs = cube_frusta()
    ffs = ffs[:3]
    view = ob.look_at_rh((0, 0, 0), (1, 0, 0), (0, -1, 0))
    vp = fb.mat4_mul(ob.perspective(1.0, float(np.pi / 2), 0.01, 120.0), view)
    out = {}

    ctx = fb.Context(device=0)
    ctx.enable_instances(True)
    # topology, then a topology change that carries the local matrices, TRS records, statics, bundle ids and LOD ranges
    first = flags.copy()
    first[late] &= ~np.uint32(fb.NODE_ALIVE)
    ctx.set_topology(sc.parent, first, sc.render_mask, aabb, root=0)
    ctx.set_local_matrices(sc.local_m16)
    statics = np.zeros((len(statics_nodes), 25), f32)
    statics[:, 3] = 1.0
    statics[:, 4] = statics[:, 8] = statics[:, 12] = 1.0
    statics[:, 13:25] = rng.uniform(-0.5, 0.5, (len(statics_nodes), 12))
    ctx.set_transform_statics(statics, statics_nodes)
    trs = np.zeros((len(lights), 10), f32)
    trs[:, 0:3] = rng.uniform(-30, 30, (len(lights), 3))
    q = rng.normal(size=(len(lights), 4)).astype(f32)
    trs[:, 3:7] = q / np.linalg.norm(q, axis=1, keepdims=True)
    trs[:, 7:10] = rng.uniform(0.5, 2.0, (len(lights), 3))
    ctx.set_local_trs(trs, lights)
    ctx.set_bundle_ids(rng.integers(0, 40, n).astype(np.uint32))
    ctx.set_lod_ranges(np.tile(np.array([0.0, 0.3], f32), (len(lod), 1)), lod)
    ctx.set_topology(sc.parent, flags, sc.render_mask, aabb, root=0)
    ctx.set_local_matrices(sc.local_m16[late], late)

    # skinned surfaces with blend shapes; the bone tables and vertex streams grow under reserve_skinning and by themselves
    ctx.reserve_skinning(2 * sc.bones_per_unit, 2 * VERTS)
    sids = []
    for u in range(sc.n_units):
        verts, _ = sc.unit_vertices(u)
        sids.append(ctx.add_skinned_surface(sc.unit_mesh_node(u), sc.unit_bone_nodes(u), sc.unit_inv_bind(u), verts))
        if u == sc.n_units // 2:
            ctx.reserve_skinning(sc.n_units * sc.bones_per_unit, sc.n_units * VERTS + 4096)
    for u in (1, 5):
        off = (rng.normal(size=(2, VERTS, 9)) * 0.2).astype(np.float16)
        ctx.set_blend_shapes(sids[u], off.view(np.uint16), np.array([40.0, 75.0], f32))
    ctx.set_node_surfaces([sc.unit_mesh_node(u) for u in range(sc.n_units)], [[(3, sids[u]), (7, None)] for u in range(sc.n_units)])

    # animations, cleared and added again
    anims = [_position_animation(pick[322 + 10 * k: 332 + 10 * k], rng) for k in range(2)]
    for t, k in anims:
        ctx.anim_add(t, k, time_slice=(0.0, 1.0))
    ctx.animate(0.25)
    ctx.anim_clear()
    for t, k in anims:
        ctx.anim_add(t, k, time_slice=(0.0, 1.0), speed=1.5)

    # LOD ranges with observers, the light lists and the reflection probes
    ctx.set_observers([((0, 0, 0), 0.1, 80.0), ((10, 0, 0), 0.1, 60.0), ((0, 5, -5), 0.5, 120.0)])
    ctx.update_and_cull(ffs, fb.UPDATE_ALL)
    ctx.cull_lights()
    for f in range(len(ffs)):
        out[f"lod_visible{f}"] = np.sort(ctx.get_visible(f))  # the cull's compaction leaves the order undefined
        out[f"lights{f}"] = ctx.get_visible_lights(f)
    out["probes"] = ctx.select_reflection_probes()
    ctx.set_observers([])

    # a synchronous frame with animation, then the shadow casters of its lights read back on the host
    ctx.render_prep(update_flags=fb.UPDATE_ALL, frusta=ffs, animate_dt=0.1)
    rec = np.zeros(len(lights), fb.Context.LIGHT_SOURCE_DTYPE)
    rec["kind"] = np.where(np.arange(len(lights)) % 2, fb.LIGHT_POINT, fb.LIGHT_SPOT)
    rec["full_cone_angle"], rec["distance_or_radius"] = 1.2, 15.0
    ctx.set_light_sources(rec, lights)
    ctx.cull_shadow_casters(0, np.zeros(3, f32), 40.0, 40.0)
    maps, entries = ctx.get_shadow_maps()
    out["shadow_maps"] = maps
    out["shadow_entries"] = np.concatenate([np.sort(entries[m["first"]: m["first"] + m["count"]]) for m in maps])

    # instances and their bone-matrix blocks read back on the host
    inst = ctx.pack_instances(0, view, vp)
    order = np.lexsort((inst["surface"], inst["node"]))  # the order inside a bundle is undefined
    out.update({f"inst_{k}": v if k == "bundles" else v[order] for k, v in inst.items()})
    ctx.pack_bone_matrices(0)
    skinned = [int(i) for i in order if int(inst["node"][i]) in units][:6]
    blocks = [ctx.get_bone_matrix_block(0, i) for i in skinned]
    out["bone_blocks"] = np.stack([np.full((255, 16), np.nan, f32) if b is None else b for b in blocks])
    assert any(b is not None for b in blocks)

    # two pipelined frames
    idx, m = sc.animate(1)
    ctx.render_prep(changed_m16=m, changed_idx=idx, frusta=ffs, async_=True, animate_dt=0.05)
    idx, m = sc.animate(2)
    ctx.render_prep(changed_m16=m, changed_idx=idx, frusta=ffs, async_=True)
    for k in range(2):
        ctx.frame_wait()
        for f in range(len(ffs)):
            out[f"frame{k}_visible{f}"] = np.sort(ctx.get_visible(f))

    # the get_* read-backs
    out["global"] = ctx.get_global_matrices()
    out["aabb"] = ctx.get_world_aabbs()
    out["flags"] = ctx.get_global_flags()
    out["anim_time"] = ctx.anim_time_positions(0, 2)
    for u, sid in enumerate(sids):
        out[f"palette{u}"] = ctx.get_palette(sid)
        out[f"pos{u}"], out[f"nrm{u}"] = ctx.get_skinned(sid)
    ctx.close()
    sc.close()

    assert len(maps) and entries.size and inst["node"].size and skinned and out["frame1_visible0"].size
    return out


def test_every_feature_then_destroy():
    first = _every_feature_round()
    for _ in range(2):
        again = _every_feature_round()
        assert again.keys() == first.keys()
        for k, v in first.items():
            assert again[k].tobytes() == v.tobytes(), k


VARIANTS = {"peer_seg": ("peer", "1"), "nccl_seg": ("nccl", "1"), "peer_private": ("peer", "0"), "nccl_private": ("nccl", "0")}


@pytest.mark.parametrize("variant", sorted(VARIANTS))
def test_single_rank_exchange_lifecycle(monkeypatch, variant):
    """World size 1: the gathered lists are the rank's own lists and the oracle's sets, whichever exchange was asked for."""
    import torch  # noqa: F401  (its NCCL is the libnccl.so.2 that fyx_comm_init binds)

    ex, hs = VARIANTS[variant]
    monkeypatch.setenv("FYX_EXCHANGE", ex)
    monkeypatch.setenv("FYX_HOSTSEG", hs)
    sc = Scene(N_NODES, n_units=N_UNITS, verts_per_unit=64)
    og = ob.Graph.build(sc.parent, sc.flags, sc.render_mask, sc.local_m16, sc.local_aabb.copy())
    for u in range(sc.n_units):
        og.add_surface(sc.unit_mesh_node(u), sc.unit_bone_nodes(u))
    og.L.orc_graph_drop_messages(og.h)
    og.update_hierarchical_data()
    fos, ffs = cube_frusta()
    want = [np.sort(og.from_graph(fo)) for fo in fos]

    ctx = fb.Context(device=0)
    try:
        ctx.set_topology(sc.parent, sc.flags, sc.render_mask, sc.local_aabb, root=0)
        ctx.set_local_matrices(sc.local_m16)
        for u in range(sc.n_units):
            verts, _ = sc.unit_vertices(u)
            ctx.add_skinned_surface(sc.unit_mesh_node(u), sc.unit_bone_nodes(u), sc.unit_inv_bind(u), verts)

        def check():
            for f in range(len(ffs)):
                gathered = np.sort(ctx.get_visible_gathered(f))
                assert np.array_equal(gathered, want[f]), (f, gathered.size, want[f].size)
                assert np.array_equal(np.sort(ctx.get_visible(f)), want[f]), f
                assert ctx.get_visible_gathered_device(f)[1] == want[f].size
            mode = ctx.comm_mode()
            assert ("peer stores" in mode) == (ex == "peer"), mode
            assert ("host segment" in mode) == (hs == "1"), mode

        ctx.comm_init(1, 0, fb.Context.comm_unique_id())
        ctx.render_prep(update_flags=fb.UPDATE_ALL, frusta=ffs, readback_visible=False, allgather=True)
        check()
        ctx.render_prep(update_flags=fb.UPDATE_ALL, frusta=ffs, readback_visible=True, allgather=True)
        check()
        for k in range(3):
            ctx.render_prep(update_flags=fb.UPDATE_ALL, frusta=ffs, readback_visible=True, allgather=True, async_=True)
            if k:
                ctx.frame_wait()
        ctx.frame_wait()
        check()
        ctx.comm_init(1, 0, fb.Context.comm_unique_id())  # tears the exchange down and starts over
        ctx.render_prep(update_flags=fb.UPDATE_ALL, frusta=ffs, readback_visible=True, allgather=True)
        check()
    finally:
        ctx.close()
        sc.close()
