"""The edge cases of tests/anim_edges.py on the device, through the C ABI: curve values at keys, one ulp either side,
t rounding to 1, duplicate keys, one-ulp spans, large locations, every kind pair and 0 to 70 000 keys; hint sequences;
time advance on inexact, empty and point slices; Euler angles up to 1e6; and the state a frame carries (animations and
blend groups added between frames, anim_clear, grid tails, a node driven by a player and a blend group in one frame).

A curve value is observed through one depth-1 node per probe under an identity root, unit scale, no statics: the
sampled position is the node's global translation, a sampled rotation its rotation block.  Each probe time is its own
animation (speed 0, clamped to a slice wide enough to hold it), so one `animate` reads hundreds of probes.  Values
equal the oracle bit for bit and the float32 restatement of anim_edges.py; Vector3 and UnitQuaternion values are within
the float64 bounds stated there; Euler rotations are within 2e-6 of the oracle (libm) and within EULER_MAT_BOUND of the
float64 rotation matrix."""
import numpy as np
import pytest

import anim_edges as ae
import fyrox_b200 as fb
import oracle_binding as ob
from helpers import NONE, assert_same_hierarchy, bits_equal
from test_gpu_anim import Builder, load_pair, make_graph, times_equal

pytestmark = pytest.mark.gpu

f32 = np.float32
TD = ob.TRACK_DTYPE
WIDE = (-3e38, 3e38)
ROT = [0, 1, 2, 4, 5, 6, 8, 9, 10]


def flat_scene(ctx, n_probes):
    n = n_probes + 1
    parent = np.full(n, NONE, np.uint32)
    parent[1:] = 0
    flags = np.full(n, fb.NODE_DEFAULT | fb.NODE_RENDERABLE, np.uint32)
    flags[0] = fb.NODE_DEFAULT
    trs = np.zeros((n, 10), np.float32)
    trs[:, 6] = trs[:, 7:10] = 1.0
    return load_pair(ctx, parent, flags, trs)


def track(node, binding, kind, curves):
    """One track whose curve c is keys[first[c] : first[c] + n[c]]."""
    t = np.zeros(1, TD)
    t[0]["target_node"], t[0]["binding"], t[0]["value_kind"], t[0]["enabled"], t[0]["n_curves"] = node, binding, kind, 1, len(curves)
    for c, (f, k) in enumerate(curves):
        t[0]["first_key"][c], t[0]["n_keys"][c] = f, k
    return t


def probe_track(node, kind, keys_list):
    """Curves of one probe, concatenated: Vector3 position (x = the curve, y = z = empty), or 3 / 4 curves."""
    keys = np.concatenate(keys_list) if keys_list else np.zeros(0, ob.KEY_DTYPE)
    curves, f = [], 0
    for k in keys_list:
        curves.append((f, len(k)))
        f += len(k)
    if kind == ob.TV_VECTOR3 and len(curves) == 1:
        curves += [(f, 0), (f, 0)]
    binding = ob.BIND_POSITION if kind == ob.TV_VECTOR3 else ob.BIND_ROTATION
    return track(node, binding, kind, curves), keys


def run_probes(ctx, probes):
    """probes = [(kind, [keys per curve], time)]; one animation per probe on node i + 1.  Returns the device's global
    matrices (after the hierarchy matched the oracle, bit for bit except Euler rotation entries)."""
    og, tr = flat_scene(ctx, len(probes))
    anims = []
    for i, (kind, keys_list, time) in enumerate(probes):
        t, k = probe_track(i + 1, kind, keys_list)
        kw = dict(speed=0.0, looped=False, time_slice=WIDE, time_position=float(time))
        anims.append(ob.Animation(t, k, **kw))
        ctx.anim_add(t, k, **kw)
    ob.update_animations(anims, 0.0, og, tr)
    og.update()
    ctx.animate(0.0)
    ctx.update_transforms(fb.UPDATE_INCREMENTAL)
    times_equal(ctx, anims)
    G, Go = ctx.get_global_matrices(), og.global_transforms()
    euler = np.array([False] + [kind == ob.TV_QUAT_EULER for kind, _, _ in probes])
    assert bits_equal(G[~euler], Go[~euler]).all(), np.nonzero(~bits_equal(G, Go).all(1) & ~euler)[0][:10]
    if euler.any():
        assert np.abs(G[euler][:, ROT] - Go[euler][:, ROT]).max() <= 2e-6
        assert bits_equal(G[euler][:, 12:16], Go[euler][:, 12:16]).all()
    ctx.anim_clear()
    return G


def test_curve_values_at_the_edges_match_oracle_and_float64(ctx):
    cases = ae.curve_cases(np.random.default_rng(9001))
    probes, want, classes = [], [], []
    for cls, cs in cases.items():
        for keys, xs in cs:
            for x in xs:
                v = ae.curve_value_at(keys, x)[0]
                if not np.isfinite(v):
                    continue  # an infinite translation is not an affine matrix: the CPU file compares these with the oracle
                probes.append((ob.TV_VECTOR3, [keys], x))
                want.append((keys, x))
                classes.append(cls)
    assert len(probes) > 600 and set(classes) == set(ae.CURVE_CLASSES)
    G = run_probes(ctx, probes)
    worst, checked = 0.0, 0
    for i, (keys, x) in enumerate(want):
        got = G[i + 1, 12]
        assert ae.same_bits(got, ae.curve_value_at(keys, x)[0]), (classes[i], x)
        v64, bound = ae.curve_value_at64(keys, x)
        if bound is not None:
            err = abs(float(got) - v64)
            assert err <= bound, (classes[i], x, got, v64, bound)
            worst = max(worst, err / bound if bound else 0.0)
            checked += 1
    print(f"curve probes: {len(probes)}, float64-checked {checked}, largest error / bound {worst:.3f}")


def test_quaternion_and_euler_tracks_match_oracle_and_float64(ctx):
    rng = np.random.default_rng(77)
    probes, info = [], []
    for _ in range(150):
        ks = [ae.random_curve(rng, int(rng.integers(2, 9)), kinds=(ae.LIN, ae.CUB)) for _ in range(4)]
        ks[3]["value"] = np.abs(ks[3]["value"]) + f32(0.5)  # keep the quaternion away from 0
        x = f32(rng.uniform(-3.2, 3.2))
        probes.append((ob.TV_QUAT, ks, x))
        info.append(("quat", ks, x))
    for cls, es in ae.euler_cases(np.random.default_rng(6)).items():
        for e in es:
            probes.append((ob.TV_QUAT_EULER, [ae.keys_of([(0.0, a, ae.CONST)]) for a in e], 0.5))
            info.append((cls, e, None))
    G = run_probes(ctx, probes)
    worst_q = worst_e = 0.0
    for i, (cls, a, x) in enumerate(info):
        R = G[i + 1, ROT].astype(np.float64)
        if cls == "quat":
            vb = [ae.curve_value_at64(k, x) for k in a]
            v64 = np.array([v for v, _ in vb])
            N = float(np.linalg.norm(v64))
            bound = 2 * sum(b for _, b in vb) / N + ae.EULER_MAT_BOUND
            err = np.abs(R - ae.rotation_matrix64(v64 / N)).max()
            assert err <= bound, (i, err, bound)
            worst_q = max(worst_q, err / bound)
        else:
            err = np.abs(R - ae.rotation_matrix64(ae.quat_from_euler64(a))).max()
            assert err <= ae.EULER_MAT_BOUND, (cls, a, err)
            worst_e = max(worst_e, err / ae.EULER_MAT_BOUND)
    print(f"rotation probes: quaternion largest error / bound {worst_q:.3f}, euler {worst_e:.3f}")


def test_hint_sequences_match_oracle_after_every_step(ctx):
    cases = ae.hint_cases(np.random.default_rng(9002))
    seqs = [(cls, keys, ts) for cls, cs in cases.items() for keys, ts in cs]
    og, tr = flat_scene(ctx, len(seqs))
    anims = []
    for i, (cls, keys, ts) in enumerate(seqs):
        t, k = probe_track(i + 1, ob.TV_VECTOR3, [keys])
        kw = dict(speed=0.0, looped=False, time_slice=WIDE, time_position=float(ts[0]))
        anims.append(ob.Animation(t, k, **kw))
        ctx.anim_add(t, k, **kw)
    hints = [0] * len(seqs)
    for step in range(max(len(ts) for _, _, ts in seqs)):
        for i, (cls, keys, ts) in enumerate(seqs):
            if 0 < step < len(ts):
                ob.lib().orc_animation_set_time_position(anims[i].h, float(ts[step]))
                ctx.anim_set_time_position(i, float(ts[step]))
        ob.update_animations(anims, 0.0, og, tr)
        og.update()
        ctx.animate(0.0)
        ctx.update_transforms(fb.UPDATE_INCREMENTAL)
        assert_same_hierarchy(og, ctx)
        G = ctx.get_global_matrices()
        for i, (cls, keys, ts) in enumerate(seqs):
            v, hints[i] = ae.curve_value_at(keys, ts[min(step, len(ts) - 1)], hints[i])
            assert ae.same_bits(G[i + 1, 12], v), (cls, step)


def test_time_advance_matches_oracle_after_every_tick(ctx):
    cases = ae.time_cases()
    parent = np.array([NONE, 0], np.uint32)
    ctx.set_topology(parent)
    empty_t, empty_k = np.zeros(0, TD), np.zeros(0, ob.KEY_DTYPE)
    anims = []
    for cls, name, (lo, hi), looped, t0, s in cases:
        kw = dict(speed=float(s), looped=looped, time_slice=(float(lo), float(hi)), time_position=float(t0))
        anims.append(ob.Animation(empty_t, empty_k, **kw))
        ctx.anim_add(empty_t, empty_k, **kw)
    times_equal(ctx, anims)
    tr = (ob.Transform * 2)()
    og = ob.Graph.build(parent, None, None, np.tile(np.eye(4, dtype=np.float32).reshape(16), (2, 1)), None)
    mine = [f32(a.time_position) for a in anims]
    for dt in (1.0, 1.0, 0.0, 1.0, 0.37, -2.5):
        ob.update_animations(anims, dt, og, tr)
        ctx.animate(dt)
        times_equal(ctx, anims)
        got = ctx.anim_time_positions(0, len(anims))
        for i, (cls, name, (lo, hi), looped, t0, s) in enumerate(cases):
            n = f32(mine[i] + f32(f32(dt) * s))
            mine[i] = ae.wrapf(n, lo, hi) if looped else min(max(n, lo), hi)
            assert ae.same_bits(got[i], mine[i]), (cls, name, looped, dt)


def _frame(ctx, og, tr, direct, groups, dt):
    ob.update_animations(direct, dt, og, tr)
    for srcs, w in groups:
        ob.blend_group_update(srcs, w, dt, og, tr)
    og.update()
    ctx.animate(dt)
    ctx.update_transforms(fb.UPDATE_INCREMENTAL)
    assert_same_hierarchy(og, ctx)


def test_animations_and_groups_added_between_frames_and_after_clear(ctx):
    rng = np.random.default_rng(31)
    n = 400
    parent, flags, trs = make_graph(rng, n)
    og, tr = load_pair(ctx, parent, flags, trs)

    def add(nodes, **kw):
        b = Builder(rng)
        for node in nodes:
            b.track(node, ob.BIND_POSITION, ob.TV_VECTOR3, key_range=(2, 30))
            b.track(node, ob.BIND_ROTATION, ob.TV_QUAT, lo=-1.0, hi=1.0, key_range=(2, 30))
        t, k = b.arrays()
        ctx.anim_add(t, k, **kw)
        return ob.Animation(t, k, **kw)

    anims = [add(range(1, 120), speed=1.0, looped=True, time_slice=(0.1, 0.7), time_position=0.3),
             add(range(80, 200), speed=-0.6, looped=False, time_slice=(-1 / 3, 5 / 7), time_position=0.5)]
    dts = [0.13, 0.3, 0.07]
    for f in range(3):
        _frame(ctx, og, tr, anims, [], dts[f])
        times_equal(ctx, anims)
    # more animations after frames: the device tables grow, the older hints and times carry over
    anims += [add(range(150, 260), speed=2.0, looped=True, time_slice=(0.0, 1.7), time_position=0.9),
              add(range(240, 330), speed=1.0, looped=True, time_slice=(0.25, 2.0), time_position=0.0),
              add(range(280, 360), speed=0.5, looped=True, time_slice=(0.0, 2.5), time_position=1.0)]
    for f in range(3):
        _frame(ctx, og, tr, anims, [], dts[f])
        times_equal(ctx, anims)
    # blend groups made after frames: sources whose node sets differ (and overlap a direct animation's), and a group
    # whose first source is disabled before its first tick, so it has no pose to clone
    anims += [add(range(330, 380), speed=1.0, looped=True, time_slice=(0.0, 2.0), time_position=0.4, enabled=False),
              add(range(340, 390), speed=1.0, looped=True, time_slice=(0.0, 2.0), time_position=0.6)]
    w1, w2 = [1.0, -0.5], [0.3, 1.0]
    assert ctx.anim_blend_group([3, 4], w1) == 1
    assert ctx.anim_blend_group([5, 6], w2) == 2
    for f in range(6):
        if f == 2:
            w1 = [0.0, 2.0]
            ctx.anim_set_blend_weights(1, w1)
        if f == 4:
            ob.lib().orc_animation_set_enabled(anims[5].h, 1)
            ctx.anim_set_enabled(5, True)
        _frame(ctx, og, tr, anims[:3], [([anims[3], anims[4]], w1), ([anims[5], anims[6]], w2)], dts[f % 3])
        times_equal(ctx, anims)
    # anim_clear, then new animations: the nodes keep the transforms the old ones left
    ctx.anim_clear()
    anims = [add(range(100, 380), speed=1.0, looped=True, time_slice=(0.0, 2.0), time_position=0.2)]
    for f in range(3):
        _frame(ctx, og, tr, anims, [], dts[f])
        times_equal(ctx, anims)


@pytest.mark.parametrize("n_anims,n_tracks", [(255, 1), (256, 1), (257, 1), (600, 1), (1, 257)])
def test_grid_tails_of_animations_and_tracks(ctx, n_anims, n_tracks):
    rng = np.random.default_rng(n_anims * 7 + n_tracks)
    n = n_anims * n_tracks + 1
    parent, flags, trs = make_graph(rng, n, depth1=True)
    og, tr = load_pair(ctx, parent, flags, trs)
    anims = []
    for a in range(n_anims):
        b = Builder(rng)
        for j in range(n_tracks):
            b.track(1 + a * n_tracks + j, ob.BIND_POSITION, ob.TV_VECTOR3, key_range=(1, 12))
        t, k = b.arrays()
        kw = dict(speed=float(rng.uniform(-2, 2)), looped=bool(a % 3), time_slice=(0.0, 2.0), time_position=float(rng.uniform(0, 2)))
        anims.append(ob.Animation(t, k, **kw))
        ctx.anim_add(t, k, **kw)
    for dt in (0.1, 0.45, 0.3):
        _frame(ctx, og, tr, anims, [], dt)
        times_equal(ctx, anims)


def test_player_and_group_on_one_node_share_the_frame_dirty_flag(ctx):
    """The player's +0 scale leaves the transform dirty, so the group's -0 is stored (scene/transform.rs:249-260; the
    player and the machine run in one Graph::update node loop with no matrix() between them)."""
    parent, trs, (td, kd), (tg, kg) = ae.zero_scale_pair()
    flags = np.full(3, fb.NODE_DEFAULT | fb.NODE_RENDERABLE, np.uint32)
    og, tr = load_pair(ctx, parent, flags, trs)
    direct, src = ob.Animation(td, kd, time_slice=(0.0, 1.0)), ob.Animation(tg, kg, time_slice=(0.0, 1.0))
    ctx.anim_add(td, kd, time_slice=(0.0, 1.0))
    ctx.anim_add(tg, kg, time_slice=(0.0, 1.0))
    ctx.anim_blend_group([1], [1.0])
    for dt in (0.1, 0.2):
        _frame(ctx, og, tr, [direct], [([src], [1.0])], dt)
        times_equal(ctx, [direct, src])
    assert np.signbit(ctx.get_global_matrices()[2, 0])
