"""The cascaded-shadow-map oracle (tests/csm_oracle.py) on hand-checked cases: the split distances of both modes and the
MIN_DEPTH_DELTA guard, the camera projections' guards (z_far < z_near, tiny and negative vertical sizes, h = 0), the
look_at_lh rows, the try_normalize fallbacks, each z_mult sign branch, the gates of light.rs:555-565, and the ABI structs."""
import ctypes as C

import numpy as np

import csm_oracle as co
import oracle_binding as ob
import shadow_oracle as so
from fyrox_b200 import _lib as L
from test_shadow_oracle_cpu import DEF, LIGHT, camera, scene

f32 = np.float32
EPS = f32(1.1920929e-07)
VIEW = ob.look_at_rh((0, 0, 0), (0, 0, -1), (0, 1, 0))


def persp(z_near=0.1, z_far=150.0, frame=(1920.0, 1080.0)):
    return co.CsmCamera(co.PERSPECTIVE, float(np.deg2rad(60.0)), z_near, z_far, frame, VIEW)


def ortho(size, z_near=0.1, z_far=150.0, frame=(1920.0, 1080.0)):
    return co.CsmCamera(co.ORTHOGRAPHIC, size, z_near, z_far, frame, VIEW)


def test_relative_eq():
    assert co.relative_eq(1.0, 1.0) and co.relative_eq(np.inf, np.inf)
    assert not co.relative_eq(np.inf, 1.0) and not co.relative_eq(1.0, -np.inf)
    assert co.relative_eq(0.0, 1e-7)  # |a - b| <= EPSILON
    assert not co.relative_eq(0.0, 2e-7)
    assert co.relative_eq(1e6, 1e6 + 0.0625)  # 0.0625 <= 1e6 * EPSILON = 0.119
    assert not co.relative_eq(1e6, 1e6 + 0.25)
    assert not co.relative_eq(np.nan, np.nan)


def test_split_distances_absolute_relative_and_the_min_depth_delta():
    cam = persp(z_near=0.1, z_far=100.0)
    absolute = [co.cascade_depths(cam, co.CSM_DEFAULT, i) for i in range(3)]
    assert absolute == [(f32(0.1), f32(5.0)), (f32(5.0), f32(25.0)), (f32(25.0), f32(64.0))]
    relative = [co.cascade_depths(cam, (1, (0.1, 0.5, 1.0)), i) for i in range(3)]
    assert relative == [(f32(0.1), f32(100.0) * f32(0.1)), (f32(100.0) * f32(0.1), f32(50.0)), (f32(50.0), f32(100.0))]
    # a split equal to z_near: z_far += (2 * EPSILON) * z_near
    zn, zf = co.cascade_depths(cam, (0, (0.1, 30.0, 40.0)), 0)
    assert zn == f32(0.1) and zf == f32(0.1) + f32(2.0) * EPS * f32(0.1) and zf > zn
    # equal far planes further out: relatively equal too
    zn, zf = co.cascade_depths(cam, (0, (5.0, 5.0, 40.0)), 1)
    assert zf == f32(5.0) + f32(2.0) * EPS * f32(5.0)


def test_slice_centers_of_a_perspective_camera():
    # looking down -Z from the origin: the slice [0.1, 5] spans z = -0.1 .. -5, its corner mean is -2.55 on the axis
    corners = co.slice_corners(persp(), f32(0.1), f32(5.0))
    c = co.frustum_center(corners)
    assert abs(c[0]) < 1e-5 and abs(c[1]) < 1e-5 and abs(c[2] + 2.55) < 1e-4
    assert np.allclose(sorted(set(np.round(corners[:, 2], 4))), [-5.0, -0.1])


def test_projection_guards():
    cam = persp()
    # z_far < z_near: the projection swaps them
    assert co.projection_matrix(cam, 10.0, 2.0).tobytes() == co.projection_matrix(cam, 2.0, 10.0).tobytes()
    # planes closer than 10 * EPSILON are pushed apart by that limit
    p = co.projection_matrix(cam, 1.0, 1.0)
    assert p[10] == (f32(1.0) + co.LIMIT + f32(1.0)) / (f32(1.0) - (f32(1.0) + co.LIMIT))
    # perspective: m22 / aspect
    p = co.projection_matrix(cam, 1.0, 10.0)
    assert p[5] == co.m22_of(np.deg2rad(60.0)) and p[0] == p[5] / (f32(1920.0) / f32(1080.0)) and p[11] == -1.0 and p[15] == 0.0
    # h = 0: aspect = inf, m22 / inf = 0
    with np.errstate(all="ignore"):
        assert co.projection_matrix(persp(frame=(640.0, 0.0)), 1.0, 10.0)[0] == 0.0
        # w = h = 0: NaN aspect, f32::max gives the limit
        assert co.projection_matrix(persp(frame=(0.0, 0.0)), 1.0, 10.0)[0] == p[5] / co.LIMIT
    # orthographic: vertical sizes clamped away from zero with their sign, horizontal = aspect * vertical
    o = co.projection_matrix(ortho(8.0, frame=(200.0, 100.0)), 1.0, 10.0)
    assert o[5] == f32(2.0) / f32(16.0) and o[0] == f32(2.0) / f32(32.0) and o[12] == 0.0 and o[15] == 1.0
    assert co.projection_matrix(ortho(1e-7), 1.0, 10.0)[5] == f32(2.0) / (co.LIMIT + co.LIMIT)
    assert co.projection_matrix(ortho(-1e-7), 1.0, 10.0)[5] == f32(2.0) / (-co.LIMIT - co.LIMIT)
    assert co.projection_matrix(ortho(-8.0, frame=(200.0, 100.0)), 1.0, 10.0)[5] == f32(2.0) / f32(-16.0)
    assert co.projection_matrix(ortho(0.0), 1.0, 10.0)[5] == f32(2.0) / (co.LIMIT + co.LIMIT)


def test_look_at_lh():
    # toward +Z with y up: the identity rotation, translation -eye
    v = co.look_at_lh((1.0, 2.0, 3.0), (1.0, 2.0, 4.0), (0.0, 1.0, 0.0))
    want = np.eye(4, dtype=f32).reshape(16).copy()
    want[12:15] = (-1.0, -2.0, -3.0)
    assert v.tobytes() == want.tobytes()
    # toward -Y with z up (the default light of a directional light: up = y, so light_direction = -y, look = z)
    v = co.look_at_lh((0.0, 1.0, 0.0), (0.0, 0.0, 0.0), (0.0, 0.0, 1.0))
    f, s = (0.0, -1.0, 0.0), (1.0, 0.0, 0.0)  # f = target - eye; s = up x f = (0,0,1) x (0,-1,0)
    assert tuple(v[[2, 6, 10]]) == f and tuple(v[[0, 4, 8]]) == s and tuple(v[[1, 5, 9]]) == (0.0, 0.0, 1.0)  # u = f x s
    assert v[14] == 1.0 and v[15] == 1.0


def test_zero_length_up_and_look_fall_back_to_y_and_z():
    cam = persp()
    got = co.cascades(cam, co.CSM_DEFAULT, np.zeros(3, f32), np.zeros(3, f32))
    want = co.cascades(cam, co.CSM_DEFAULT, np.array([0, 1, 0], f32), np.array([0, 0, 1], f32))
    for (v, vp), (wv, wvp) in zip(got, want):
        assert v.tobytes() == wv.tobytes() and vp.tobytes() == wvp.tobytes()
    assert len(got) == 3


def test_z_mult_sign_branches():
    assert co.z_stretch(f32(-2.0), f32(3.0)) == (f32(-20.0), f32(30.0))
    assert co.z_stretch(f32(2.0), f32(3.0)) == (f32(0.2), f32(30.0))
    assert co.z_stretch(f32(-2.0), f32(-1.0)) == (f32(-20.0), f32(-0.1))
    assert co.z_stretch(f32(0.0), f32(-0.0)) == (f32(0.0), f32(-0.0))  # 0 is not < 0: divided / multiplied


def test_cascade_boxes_hold_their_slice():
    cam = persp()
    for i, (v, vp) in enumerate(co.cascades(cam, co.CSM_DEFAULT, np.array([0.3, 1.0, 0.2], f32), np.array([0, 0, 1], f32))):
        corners = co.slice_corners(cam, *co.cascade_depths(cam, co.CSM_DEFAULT, i))
        fr = ob.frustum_from_vp(vp)
        assert fr is not None
        for c in corners:  # every corner of the slice lies in the cascade's box (x, y exactly on its faces at worst)
            p = co.transform_point(vp, c)
            assert np.all(np.abs(p) <= 1.0 + 1e-5), (i, p)


def sun(flags=DEF | LIGHT, scale=None):
    m = ob.translation(0.0, 0.0, -3.0)
    if scale is not None:
        m = ob.mat4_mul(m, ob.scaling(*scale))
    og, fl = scene(m, light_flags=flags)
    return og, fl


def maps(og, flags, csm, scale=None):
    return co.shadow_maps(og, flags, camera(), (0.0, 0.0, 0.0), 0xFFFFFFFF, (10.0, 10.0, 1, 1), {1: (so.LIGHT_DIRECTIONAL, 0.0, 0.0)},
                          scale or {}, csm=csm)


def test_gates():
    og, flags = sun()
    got = maps(og, flags, persp())
    assert [(m[0], m[1], m[2]) for m in got] == [(1, 0, 0), (1, 0, 1), (1, 0, 2)]
    assert len(got[0][4]) > 0 and len(got[1][4]) > 0 and len(got[2][4]) == 0  # meshes at z = -4 .. -14: the first two slices
    # without csm: exactly the spot / point oracle (no maps for a directional light)
    assert maps(og, flags, None) == []
    # csm_settings.enabled = false
    off = persp()
    off.enabled = False
    assert maps(og, flags, off) == []
    # no cast_shadows
    og2, flags2 = sun(flags=(DEF | LIGHT) & ~so.NODE_CAST_SHADOWS)
    assert maps(og2, flags2, persp()) == []
    # a zero scale: radius 0 * f32::MAX = 0, so only a light inside the camera frustum passes the sphere test
    assert len(maps(og, flags, persp(), scale={1: (0.0, 0.0, 0.0)})) == 3
    # behind the camera, in the light list through a large box
    og3, flags3 = scene(ob.translation(0.0, 0.0, 3.0), light_aabb=np.array([-10, -10, -10, 10, 10, 10], f32))
    assert co.shadow_maps(og3, flags3, camera(), (0.0, 0.0, 0.0), 0xFFFFFFFF, (10.0, 10.0, 1, 1), {1: (so.LIGHT_DIRECTIONAL, 0.0, 0.0)},
                          {1: (0.0, 0.0, 0.0)}, csm=persp()) == []
    # ... while a unit scale gives an infinite radius: every light of the list passes
    assert len(co.shadow_maps(og3, flags3, camera(), (0.0, 0.0, 0.0), 0xFFFFFFFF, (10.0, 10.0, 1, 1), {1: (so.LIGHT_DIRECTIONAL, 0.0, 0.0)},
                              {}, csm=persp())) == 3


def test_struct_sizes():
    assert C.sizeof(L.fyx_csm_options) == 16
    assert C.sizeof(L.fyx_csm_camera) == 4 * 6 + 64 + 4
    assert L.fyx_csm_camera.view_matrix.offset == 24 and L.fyx_csm_camera.csm_enabled.offset == 88
