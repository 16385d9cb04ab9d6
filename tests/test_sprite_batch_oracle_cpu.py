"""The quad nodes of the push_triangles oracle (tests/dynamic_batch_oracle.py, tests/sprite_batch_oracle.py) on hand-built
passes with known answers, the record layout, and the scene mirror's quad nodes, none of which needs a GPU."""
import ctypes as C

import numpy as np
import pytest

import dynamic_batch_oracle as dbo
import sprite_batch_oracle as sbo
from fyrox_b200 import _lib as L
from fyrox_b200 import scene
from fyrox_b200.context import Context

f32 = np.float32
SPRITE_LAYOUT = (40, 0, dbo.NONE, dbo.NONE)


def ident(_):
    return np.eye(4, dtype=f32).reshape(16)


def moved(x, y, z):
    m = np.eye(4, dtype=f32)
    m[:3, 3] = (x, y, z)
    return m.T.reshape(16).copy()


def run(nodes, dyn=None, quads=None, shadow=False, cast=lambda n: True, world=ident, sort=None, n_surf=None):
    dyn = dyn or {}
    return dbo.dynamic_pass(nodes, n_surf or (lambda n: 1 + max([k for (m, k) in dyn if m == n], default=-1)), dyn,
                            sort or (lambda n: 100), world, quads, shadow, cast)


def test_record_is_48_bytes():
    class Rec(C.Structure):  # fyx_sprite as the header declares it
        _fields_ = [("kind", C.c_uint32), ("batch_key", C.c_uint32), ("layout_id", C.c_uint32), ("flip", C.c_uint32),
                    ("uv_rect", C.c_float * 4), ("size", C.c_float), ("rotation", C.c_float), ("color", C.c_uint8 * 4),
                    ("reserved", C.c_uint32)]

    assert C.sizeof(Rec) == 48 and Context.SPRITE.itemsize == 48
    for name, _ in Rec._fields_:
        assert getattr(Rec, name).offset == Context.SPRITE.fields[name][1], name


UV = (0.25, 0.5, 0.125, 0.25)  # lx 0.25, rx 0.375, ty 0.5, by 0.75
L_, R_, T_, B_ = 0.25, 0.375, 0.5, 0.75


@pytest.mark.parametrize("fx", [False, True])
@pytest.mark.parametrize("fy", [False, True])
def test_sprite_vertices_by_hand(fx, fy):
    q = sbo.Quad(sbo.SPRITE, 0, 0, UV, (10, 20, 30, 40), 1.5, 0.75, fx, fy)
    out, pushed = run([7], quads={7: q}, world=lambda n: moved(1.0, 2.0, 3.0))
    assert pushed == []
    v = out["streams"][0]["vertices"]
    assert v.size == 160 and out["streams"][0]["stride"] == 40
    rec = v.reshape(4, 40)
    fl = rec[:, :36].copy().view(f32).reshape(4, 9)
    u = [L_ if fx else R_, R_ if fx else L_, R_ if fx else L_, L_ if fx else R_]
    w = [B_ if fy else T_] * 2 + [T_ if fy else B_] * 2
    signs = [(0.5, 0.5), (-0.5, 0.5), (-0.5, -0.5), (0.5, -0.5)]
    for k in range(4):
        assert fl[k].tolist() == [1.0, 2.0, 3.0, u[k], w[k], 1.5, 0.75, *signs[k]]
        assert rec[k, 36:].tolist() == [10, 20, 30, 40]
    assert out["streams"][0]["triangles"].tolist() == [[0, 1, 2], [0, 2, 3]]
    assert out["instances"][["node", "triangle_offset", "triangle_count"]].tolist() == [(7, 0, 2)]


@pytest.mark.parametrize("fx", [False, True])
@pytest.mark.parametrize("fy", [False, True])
def test_rectangle_vertices_by_hand(fx, fy):
    q = sbo.Quad(sbo.RECTANGLE, 0, 1, UV, (1, 2, 3, 4), 9.0, 9.0, fx, fy)
    m = np.diag([2.0, 4.0, 1.0, 1.0]).astype(f32)
    m[:3, 3] = (10.0, 20.0, 30.0)
    out, _ = run([3], quads={3: q}, world=lambda n: m.T.reshape(16).copy())
    rec = out["streams"][1]["vertices"].reshape(4, 24)
    fl = rec[:, :20].copy().view(f32).reshape(4, 5)
    u = [R_ if fx else L_, L_ if fx else R_, L_ if fx else R_, R_ if fx else L_]  # the sprite's column mirrored
    w = [B_ if fy else T_] * 2 + [T_ if fy else B_] * 2
    pos = [(11.0, 22.0), (9.0, 22.0), (9.0, 18.0), (11.0, 18.0)]
    for k in range(4):
        assert fl[k].tolist() == [*pos[k], 30.0, u[k], w[k]]
        assert rec[k, 20:].tolist() == [1, 2, 3, 4]


def test_negative_size_and_rounding_uv_sums():
    uv = (0.6, 0.3, 0.1, 0.6)  # the f32 sums 0.6 + 0.1 and 0.3 + 0.6 are not the f32 of 0.7 and 0.9
    q = sbo.Quad(sbo.SPRITE, 0, 0, uv, size=-2.5, rotation=-1.0)
    out, _ = run([1], quads={1: q})
    fl = out["streams"][0]["vertices"].reshape(4, 40)[:, :36].copy().view(f32).reshape(4, 9)
    assert fl[0, 3] == f32(0.6) + f32(0.1) and fl[0, 3] != f32(0.7)
    assert fl[2, 4] == f32(0.3) + f32(0.6) and fl[2, 4] != f32(0.9)
    assert (fl[:, 5] == f32(-2.5)).all() and (fl[:, 6] == f32(-1.0)).all()


def test_gates():
    quads = {1: sbo.Quad(sbo.SPRITE, 0, 0), 2: sbo.Quad(sbo.RECTANGLE, 1, 1), 3: sbo.Quad(sbo.SPRITE, 0, 0)}
    nodes = [1, 2, 3]
    out, pushed = run(nodes, quads=quads)
    assert out["instances"]["node"].tolist() == [1, 3, 2] and pushed == []  # 1 and 3 share a bundle: one run each
    assert out["bundles"]["count"].tolist() == [2, 1]
    # a sprite without cast_shadows is drawn in no pass; a rectangle is unaffected
    out, _ = run(nodes, quads=quads, cast=lambda n: n != 1)
    assert out["instances"]["node"].tolist() == [2, 3]
    out, pushed = run(nodes, quads=quads, shadow=True)  # nothing in a shadow pass, and no ordinary instance either
    assert out["bundles"].size == 0 and not out["streams"] and pushed == []


def test_alternating_mesh_and_sprite_pushes():
    mesh = dbo.DynSurface(5, 0, SPRITE_LAYOUT, bytes(range(120)), np.array([[0, 1, 2]], np.uint32))  # SpriteVertex layout
    nodes = [1, 2, 3, 4]
    dyn = {(1, 0): mesh, (3, 0): mesh}
    one = {2: sbo.Quad(sbo.SPRITE, 5, 0), 4: sbo.Quad(sbo.SPRITE, 5, 0)}
    out, _ = run(nodes, dyn, one)
    assert out["instances"][["node", "triangle_offset", "triangle_count"]].tolist() == [(1, 0, 6)]  # one run of all four
    st = out["streams"][0]
    assert st["vertices"].size == (3 + 4 + 3 + 4) * 40  # the mesh shares the sprites' stream
    assert st["triangles"].tolist() == [[0, 1, 2], [3, 4, 5], [3, 5, 6], [7, 8, 9], [10, 11, 12], [10, 12, 13]]
    assert st["vertices"][:120].tobytes() == bytes(range(120))  # the identity world keeps the mesh's bytes
    two = {2: sbo.Quad(sbo.SPRITE, 6, 0), 4: sbo.Quad(sbo.SPRITE, 6, 0)}
    out, _ = run(nodes, dyn, two)  # two keys: every push starts a run
    assert out["bundles"][["batch_key", "count"]].tolist() == [(5, 2), (6, 2)]
    assert out["instances"][["node", "triangle_offset", "triangle_count"]].tolist() == [(1, 0, 1), (3, 3, 1), (2, 1, 2), (4, 4, 2)]


def test_mirror_quad_nodes():
    n = scene.SpriteBuilder().with_size(5.0).with_flip_x(True)._n
    assert n.kind == "sprite" and n.flags_word() & L.NODE_RENDERABLE and n.size == f32(5.0) and n.flip_x
    assert n.local_bounding_box.tolist() == [-0.5, -0.5, -0.5, 0.5, 0.5, 0.5]  # the unit box, whatever the size
    r = scene.RectangleBuilder().with_color((1, 2, 3, 4))._n
    assert r.kind == "rectangle" and r.flags_word() & L.NODE_RENDERABLE and r.color == (1, 2, 3, 4)
    assert scene.dynamic_layout(scene.SPRITE_VERTEX_ATTRIBUTES) == (40, 0, L.FYX_NONE, L.FYX_NONE)
    assert scene.dynamic_layout(scene.RECTANGLE_VERTEX_ATTRIBUTES) == (24, 0, L.FYX_NONE, L.FYX_NONE)
