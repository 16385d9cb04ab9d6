"""The dynamic-batching oracle (tests/dynamic_batch_oracle.py) on hand-built passes with known answers, the layout rule of the
mirror, and the argument checks of the new entry points that need no GPU."""
import ctypes as C

import numpy as np

import dynamic_batch_oracle as dbo
from fyrox_b200 import scene
from fyrox_b200 import _lib as L

f32 = np.float32
NONE = dbo.NONE
LAYOUT = (48, 0, 12, 24)  # position, normal, tangent, then 8 bytes of uv


def verts(n, seed=0):
    rng = np.random.default_rng(seed)
    v = rng.standard_normal((n, 12)).astype(f32)
    return v.tobytes()


def surf(key, n=3, layout_id=0, layout=LAYOUT, seed=0):
    return dbo.DynSurface(key, layout_id, layout, verts(n, seed), np.arange(n // 3 * 3, dtype=np.uint32).reshape(-1, 3))


def ident(_):
    return np.eye(4, dtype=f32).reshape(16)


def run(nodes, dyn, n_surf=None, sort=None, world=ident):
    return dbo.dynamic_pass(nodes, n_surf or (lambda n: 1 + max([k for (m, k) in dyn if m == n], default=-1)), dyn,
                            sort or (lambda n: 100), world)


def test_identity_world_keeps_the_bytes():
    s = surf(0, 6, seed=1)
    out, _ = run([5], {(5, 0): s})
    assert out["streams"][0]["vertices"].tobytes() == s.vertices
    assert out["streams"][0]["triangles"].tolist() == s.triangles.tolist()


def test_translation_moves_positions_only_and_keeps_tangent_w():
    s = surf(0, 6, seed=2)
    m = np.eye(4, dtype=f32)
    m[:3, 3] = (1.5, -2.0, 3.25)
    out, _ = run([1], {(1, 0): s}, world=lambda n: m.T.reshape(16).copy())  # column-major
    a = np.frombuffer(s.vertices, f32).reshape(-1, 12)
    b = out["streams"][0]["vertices"].view(f32).reshape(-1, 12)
    assert np.array_equal(b[:, 0:3], a[:, 0:3] + np.array([1.5, -2.0, 3.25], f32))
    assert b[:, 3:12].tobytes() == a[:, 3:12].tobytes()  # normal, tangent xyz (a vector ignores translation), tangent w, uv


def test_rotation_turns_normals_and_tangents():
    s = surf(0, 2, seed=3)
    m = np.array([[0, -1, 0, 0], [1, 0, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]], f32)  # 90 degrees about z
    out, _ = run([1], {(1, 0): s}, world=lambda n: m.T.reshape(16).copy())
    a = np.frombuffer(s.vertices, f32).reshape(-1, 12)
    b = out["streams"][0]["vertices"].view(f32).reshape(-1, 12)
    for off in (0, 3, 6):
        assert np.array_equal(b[:, off:off + 3], np.stack([-a[:, off + 1], a[:, off], a[:, off + 2]], 1))
    assert np.array_equal(b[:, 9], a[:, 9])


def test_two_surfaces_of_one_node_in_one_bundle_are_one_instance():
    out, _ = run([3], {(3, 0): surf(7), (3, 1): surf(7, 6)})
    assert out["bundles"]["count"].tolist() == [1]
    assert out["instances"][["node", "triangle_offset", "triangle_count"]].tolist() == [(3, 0, 3)]
    assert out["streams"][0]["triangles"][1:].min() == 3  # the second surface's indices follow the first's three vertices


def test_adjacent_nodes_at_one_sort_index_are_one_instance():
    out, _ = run([1, 2], {(1, 0): surf(4), (2, 0): surf(4)})
    assert out["instances"][["node", "triangle_count"]].tolist() == [(1, 2)]


def test_a_bundle_interrupted_by_another_gives_two_instances():
    out, _ = run([1, 2, 3], {(1, 0): surf(4), (2, 0): surf(5), (3, 0): surf(4)})
    assert out["bundles"][["batch_key", "first", "count"]].tolist() == [(4, 0, 2), (5, 2, 1)]
    assert out["instances"][["node", "triangle_offset"]].tolist() == [(1, 0), (3, 2), (2, 1)]


def test_other_sort_index_is_another_bundle():
    out, _ = run([1, 2], {(1, 0): surf(4), (2, 0): surf(4)}, sort=lambda n: 10 * n)
    assert out["bundles"][["batch_key", "sort_index"]].tolist() == [(4, 10), (4, 20)]


def test_an_ordinary_push_in_between_does_not_split_a_run():
    dyn = {(1, 0): surf(4), (2, 1): surf(4)}
    out, pushed = run([1, 2], dyn, n_surf=lambda n: 2)
    assert pushed == [(1, 1), (2, 0)]
    assert out["instances"][["node", "triangle_count"]].tolist() == [(1, 2)]


def test_two_layouts_give_independent_streams():
    lay2 = (16, 0, NONE, NONE)
    s2 = dbo.DynSurface(9, 1, lay2, np.arange(12, dtype=f32).tobytes(), np.array([[2, 1, 0]], np.uint32))
    out, _ = run([1, 2, 3], {(1, 0): surf(4), (2, 0): s2, (3, 0): surf(4, 6)})
    assert sorted(out["streams"]) == [0, 1]
    assert out["streams"][1]["triangles"].tolist() == [[2, 1, 0]]
    assert out["streams"][0]["triangles"][1:].tolist() == [[3, 4, 5], [6, 7, 8]]
    assert out["instances"][["node", "triangle_offset"]].tolist() == [(1, 0), (3, 1), (2, 0)]


def test_a_random_pass_batches_or_pushes_every_surface_once():
    """Nodes of one or two surfaces, some batched under three keys, four sort indices, moved worlds: the stream is the batched
    surfaces' transformed vertices in push order with their triangles shifted, the rest are pushed, the bundles follow the first
    pushes and their instances cover every triangle."""
    rng = np.random.default_rng(3)
    dyn = {}
    for n in range(1, 40):
        for k in range(int(rng.integers(1, 3))):
            if rng.random() < 0.6:
                v = rng.standard_normal((int(rng.integers(3, 12)), 12)).astype(f32)
                dyn[(n, k)] = dbo.DynSurface(int(rng.integers(0, 3)), 0, LAYOUT, v.tobytes(), rng.integers(0, len(v), (4, 3)).astype(np.uint32))
    n_surf = {n: 1 + max([k for (m, k) in dyn if m == n], default=0) for n in range(1, 40)}
    sort = lambda n: n % 4  # noqa: E731
    world = lambda n: np.array([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, n * 0.5, -1.0, 2.0, 1], f32)  # noqa: E731
    out, pushed = run(list(range(1, 40)), dyn, n_surf=lambda n: n_surf[n], sort=sort, world=world)
    order = [(n, k) for n in range(1, 40) for k in range(n_surf[n])]
    batched = [p for p in order if p in dyn]
    assert pushed == [p for p in order if p not in dyn]
    st = out["streams"][0]
    assert st["vertices"].tobytes() == b"".join(dbo.transform_vertices(dyn[p].vertices, LAYOUT, world(p[0])) for p in batched)
    first = np.cumsum([0] + [len(dyn[p].vertices) // LAYOUT[0] for p in batched])
    assert st["triangles"].tolist() == np.concatenate([dyn[p].triangles + np.uint32(f) for p, f in zip(batched, first)]).tolist()
    keys = list(dict.fromkeys((dyn[p].batch_key, sort(p[0])) for p in batched))
    assert out["bundles"][["batch_key", "sort_index"]].tolist() == keys
    assert out["instances"]["triangle_count"].sum() == sum(len(dyn[p].triangles) for p in batched)


def test_the_mirrors_layout_rule_looks_only_at_sizes():
    # a 12-byte "position" of any declared type is transformed; a 16-byte normal, a 12-byte tangent or an 8-byte position is not
    assert scene.dynamic_layout([("position", 12), ("normal", 12), ("tangent", 16), ("uv", 8)]) == (48, 0, 12, 24)
    assert scene.dynamic_layout([("uv", 8), ("position", 12), ("normal", 16), ("tangent", 12)]) == (48, 8, NONE, NONE)
    assert scene.dynamic_layout([("position", 8)]) == (8, NONE, NONE, NONE)
    assert scene.dynamic_layout(scene.ANIMATED_VERTEX_ATTRIBUTES) == (68, 0, 20, 32)


def test_the_mirror_batches_what_the_reference_batches():
    """scene/mesh/mod.rs:739-753: a Dynamic mesh with no blend shapes on any surface; per surface no bones and < 256 vertices."""
    lay = [("position", 12)]
    mesh = scene.Node("mesh")
    mesh.surfaces = [scene.Surface(vertex_buffer=np.zeros(12 * 255, np.uint8), layout=lay),
                     scene.Surface(vertex_buffer=np.zeros(12 * 256, np.uint8), layout=lay),
                     scene.Surface(vertex_buffer=np.zeros(12 * 3, np.uint8), layout=lay, bones=[scene.Handle(1, 1)]),
                     scene.Surface(vertex_buffer=np.zeros(68 * 3, np.uint8))]
    assert mesh.batched_surfaces() == []  # BatchingMode::None
    mesh.batching_mode = scene.BatchingMode.DYNAMIC
    assert mesh.batched_surfaces() == [0, 3]
    mesh.surfaces[1].blend_shapes_container = scene.BlendShapesContainer([scene.BlendShape()])
    assert mesh.batched_surfaces() == []  # the mesh-level blend-shape test
    mesh.surfaces[1].blend_shapes_container = scene.BlendShapesContainer([])
    assert mesh.batched_surfaces() == [0, 3]
    assert scene.Node("pivot").batched_surfaces() == []


def test_struct_sizes_and_null_arguments():
    assert C.sizeof(L.fyx_dynamic_layout) == 16 and C.sizeof(L.fyx_dynamic_stream) == 32 and C.sizeof(L.fyx_dynamic_batches) == 40
    lib = L.load()
    out = L.fyx_dynamic_batches()
    for fn in ("fyx_get_dynamic_batches", "fyx_get_shadow_dynamic_batches", "fyx_get_scene_observer_dynamic_batches"):
        for suffix in ("", "_device"):
            assert getattr(lib, fn + suffix)(None, 0, C.byref(out)) == L.FYX_ERR_INVALID_ARGUMENT
    assert lib.fyx_clear_dynamic_surfaces(None, 0, None) == L.FYX_ERR_INVALID_ARGUMENT
    assert lib.fyx_add_dynamic_surface(None, 0, 0, 0, 0, None, 0, None, 0, None, None) == L.FYX_ERR_INVALID_ARGUMENT
