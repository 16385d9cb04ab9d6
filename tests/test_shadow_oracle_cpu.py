"""The shadow-map oracle (tests/shadow_oracle.py) on hand-built scenes: each gate of renderer/light.rs:509-606 on and off, the
inclusive distance bound, the cascade boundaries (a distance equal to b1 falls to cascade 2), the try_normalize fallbacks and
a scaled light; and Frustum::is_intersects_sphere against the reference's own unit test (K17)."""
import numpy as np
import pytest

import oracle_binding as ob
import shadow_oracle as so
from fyrox_b200.camera import CUBE_FACES as PRODUCT_CUBE_FACES

f32 = np.float32
DEF = 0x1F | (1 << 5)  # visibility, enabled, frustum_culling, cast_shadows, alive, renderable
LIGHT = 1 << 6


def test_k17_frustum_is_intersects_sphere():
    # fyrox-math/src/frustum.rs:540-552 (test_frustum_is_intersects_sphere)
    f = ob.frustum_from_vp(np.eye(4, dtype=np.float32).reshape(16))
    assert f is not None
    assert so.frustum_is_intersects_sphere(f, (0.0, 0.0, 0.0), 1.0)
    assert so.frustum_is_intersects_sphere(f, (0.0, 0.0, 0.0), 2.0)
    assert not so.frustum_is_intersects_sphere(f, (10.0, 10.0, 10.0), 1.0)


def test_cube_face_table_matches_the_reference_and_the_product():
    # renderer/utils.rs:49-75, in CubeMapFace order +X, -X, +Y, -Y, +Z, -Z
    want = [((1, 0, 0), (0, -1, 0)), ((-1, 0, 0), (0, -1, 0)), ((0, 1, 0), (0, 0, 1)), ((0, -1, 0), (0, 0, -1)), ((0, 0, 1), (0, -1, 0)),
            ((0, 0, -1), (0, -1, 0))]
    assert so.CUBE_FACES == want
    assert [tuple(map(tuple, fu)) for fu in PRODUCT_CUBE_FACES] == want


def camera():
    view = ob.look_at_rh((0, 0, 0), (0, 0, -1), (0, 1, 0))
    proj = ob.perspective(16 / 9, float(np.deg2rad(60.0)), 0.1, 150.0)
    return ob.frustum_from_vp(ob.mat4_mul(proj, view))


def scene(light_m16, light_flags=DEF | LIGHT, light_aabb=None):
    """root 0, light 1 (local matrix light_m16), meshes 2.. on a line in front of the camera."""
    n = 8
    parent = np.array([0xFFFFFFFF] + [0] * (n - 1), np.uint32)
    flags = np.full(n, DEF, np.uint32)
    flags[1] = light_flags
    local = np.tile(ob.translation(0, 0, 0), (n, 1))
    local[1] = light_m16
    for k in range(2, n):
        local[k] = ob.translation(0.0, 0.0, -2.0 * k)
    aabb = np.tile(np.array([-0.5, -0.5, -0.5, 0.5, 0.5, 0.5], np.float32), (n, 1))
    if light_aabb is not None:
        aabb[1] = light_aabb
    og = ob.Graph.build(parent, flags, None, local.reshape(-1), aabb.reshape(-1))
    og.update_hierarchical_data()
    return og, flags


def maps(og, flags, sources, settings=(10.0, 10.0, 1, 1), scale=None, cam_t=(0.0, 0.0, 0.0)):
    return so.shadow_maps(og, flags, camera(), cam_t, 0xFFFFFFFF, settings, sources, scale or {})


SPOT = {1: (so.LIGHT_SPOT, f32(np.deg2rad(45.0)), 4.0)}
POINT = {1: (so.LIGHT_POINT, 0.0, 3.0)}


def test_spot_and_point_counts_and_lists():
    og, flags = scene(ob.translation(0, 0, -5))
    m = maps(og, flags, SPOT)
    assert [(x[0], x[1]) for x in m] == [(1, 0)]
    assert set(m[0][4].tolist()) == set(np.sort(og.from_graph(ob.frustum_from_vp(m[0][3]), 0xFFFFFFFF, True)).tolist())
    m = maps(og, flags, POINT)
    assert [(x[0], x[1]) for x in m] == [(1, k) for k in range(6)]
    assert len({x[2] for x in m}) == 1
    # the -Z face looks along the line of meshes: a mesh within the radius is in it, one beyond the far plane is not
    assert 3 in set(m[5][4].tolist()) and 2 not in set(m[5][4].tolist()) and 7 not in set(m[5][4].tolist())
    assert maps(og, flags, {1: (so.LIGHT_DIRECTIONAL, 0.0, 3.0)}) == []
    assert maps(og, flags, {1: (so.LIGHT_UNKNOWN, 0.0, 3.0)}) == []
    assert maps(og, flags, {}) == []


@pytest.mark.parametrize("gate", ["cast_shadows", "spot_disabled", "not_a_light", "hidden", "too_far"])
def test_each_gate_removes_the_map(gate):
    light_flags = DEF | LIGHT
    settings = (10.0, 10.0, 1, 1)
    if gate == "cast_shadows":
        light_flags &= ~(1 << 3)
    if gate == "not_a_light":
        light_flags &= ~LIGHT
    if gate == "hidden":
        light_flags &= ~1
    if gate == "spot_disabled":
        settings = (10.0, 10.0, 0, 1)
    if gate == "too_far":
        settings = (4.0, 10.0, 1, 1)
    og, flags = scene(ob.translation(0, 0, -5), light_flags)
    assert len(maps(og, flags, SPOT)) == 1 or gate != "spot_disabled"  # sanity: point enabled does not matter for a spot
    assert maps(og, flags, SPOT, settings) == []
    og2, flags2 = scene(ob.translation(0, 0, -5))
    assert len(maps(og2, flags2, SPOT)) == 1


def test_distance_bound_is_inclusive():
    og, flags = scene(ob.translation(0, 0, -10))
    assert len(maps(og, flags, SPOT, (10.0, 10.0, 1, 1))) == 1
    assert maps(og, flags, SPOT, (float(np.nextafter(f32(10.0), f32(0.0))), 10.0, 1, 1)) == []


def test_sphere_gate_uses_the_light_radius():
    # the light's box reaches into the camera frustum (it is in the light list) while its centre is behind the camera
    box = np.array([-30, -30, -30, 30, 30, 30], np.float32)
    og, flags = scene(ob.translation(0, 0, 20), light_aabb=box)
    assert 1 in og.collect_lights(camera()).tolist()
    far = (100.0, 100.0, 1, 1)
    assert maps(og, flags, {1: (so.LIGHT_POINT, 0.0, 1.0)}, far) == []
    assert len(maps(og, flags, {1: (so.LIGHT_POINT, 0.0, 25.0)}, far)) == 6


@pytest.mark.parametrize("z,want", [(-9.0, 0), (-10.0, 2), (-15.0, 1), (-20.0, 2), (-25.0, 2)])
def test_cascade_boundaries(z, want):
    # shadows_distance 50: b1 = 10, b2 = 20; a distance equal to b1 is neither < b1 nor > b1 (light.rs:592-602)
    assert f32(50.0) * f32(0.2) == f32(10.0)
    og, flags = scene(ob.translation(0, 0, z))
    m = maps(og, flags, {1: (so.LIGHT_SPOT, f32(1.0), 1.0)}, (50.0, 50.0, 1, 1))
    assert [x[2] for x in m] == [want]


def test_camera_inside_the_light_radius_is_cascade_0():
    og, flags = scene(ob.translation(0, 0, -15))
    m = maps(og, flags, {1: (so.LIGHT_POINT, 0.0, 15.0)}, (50.0, 50.0, 1, 1))
    assert {x[2] for x in m} == {0}


def test_zero_up_and_look_vectors_fall_back():
    f = f32(np.deg2rad(50.0))
    pos = np.array([0.5, 0.25, -6.0], f32)
    # up vector (column 1) zero: emit direction = +Z; look vector (column 2) +X
    m16 = ob.translation(*pos)
    m16[4:7] = 0.0
    m16[8:11] = (1.0, 0.0, 0.0)
    og, flags = scene(m16)
    got = maps(og, flags, {1: (so.LIGHT_SPOT, f, 4.0)})[0][3]
    proj = ob.perspective(1.0, float(f), 0.01, 4.0)
    want = ob.mat4_mul(proj, ob.look_at_rh(pos, pos - np.array([0, 0, 1], f32), np.array([1, 0, 0], f32)))
    assert np.isfinite(want).all() and got.tobytes() == want.tobytes()
    # look vector (column 2) zero: up = +Y; up vector (0, 1, 0) is the emit direction
    m16 = ob.translation(*pos)
    m16[8:11] = 0.0
    og, flags = scene(m16)
    got = maps(og, flags, {1: (so.LIGHT_SPOT, f, 4.0)})[0][3]
    want = ob.mat4_mul(proj, ob.look_at_rh(pos, pos - np.array([0, 1, 0], f32), np.array([0, 1, 0], f32)))
    assert got.tobytes() == want.tobytes()  # emit direction and up coincide: the reference's matrix is NaN too


def test_scaled_light_scales_the_far_plane_and_the_radius():
    og, flags = scene(ob.translation(0, 0, -5))
    m = maps(og, flags, POINT, scale={1: (1.0, 3.0, 2.0)})
    proj = ob.perspective(1.0, float(so.FRAC_PI_2), 0.01, 9.0)
    pos = np.array([0, 0, -5], f32)
    look, up = so.CUBE_FACES[5]
    want = ob.mat4_mul(proj, ob.look_at_rh(pos, pos + np.array(look, f32), np.array(up, f32)))
    assert m[5][3].tobytes() == want.tobytes()
    assert 7 in set(m[5][4].tolist())  # z = -14 is 9 from the light: inside the scaled radius, outside the unscaled one
    assert 7 not in set(maps(og, flags, POINT)[5][4].tolist())
