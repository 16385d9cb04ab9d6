"""The oracle of fyx_cull_scene_observers on its own (no GPU): the order of ObserversCollection::from_scene, its gates,
Camera::calculate_matrices and the projections it uses."""
import numpy as np

import csm_oracle as co
import fyrox_b200 as fb
import observer_oracle as oo
import oracle_binding as ob
import shadow_oracle as so

f32 = np.float32
NONE = 0xFFFFFFFF


def scene():
    """root 0; 1 camera, 2 probe (Once), 3 disabled camera, 4 probe (EachFrame), 5 disabled pivot with camera 6 and probe 7
    under it, 8 probe (Once) with a rendering offset; meshes 9..14 spread around."""
    n = 15
    parent = np.zeros(n, np.uint32)
    parent[0] = NONE
    parent[6] = parent[7] = 5
    flags = np.full(n, fb.NODE_DEFAULT, np.uint32)
    flags[[2, 4, 7, 8]] |= np.uint32(fb.NODE_REFLECTION_PROBE)
    flags[5] &= ~np.uint32(fb.NODE_ENABLED)
    flags[9:] |= np.uint32(fb.NODE_RENDERABLE)
    local = np.tile(np.eye(4, dtype=f32).reshape(16), (n, 1))
    rng = np.random.default_rng(5)
    local[1:, 12:15] = rng.uniform(-5, 5, (n - 1, 3))
    local[1:, 14] -= 8.0
    aabb = np.tile(np.array([-1, -1, -1, 1, 1, 1], f32), (n, 1))
    mask = np.full(n, 0xFFFFFFFF, np.uint32)
    og = ob.Graph.build(parent, flags, mask, local, aabb)
    og.update_hierarchical_data()
    cams = {1: oo.Camera(), 3: oo.Camera(enabled=False), 6: oo.Camera()}
    probes = {2: oo.Probe(), 4: oo.Probe(update_mode=oo.EACH_FRAME), 7: oo.Probe(), 8: oo.Probe(rendering_position=(0.5, -1.0, 2.0))}
    return og, mask, cams, probes


def keys(obs):
    return [(o["node"], o["kind"], o["face"]) for o in obs]


def test_order_and_gates_across_calls():
    og, mask, cams, probes = scene()
    st = oo.ProbeState()
    faces = lambda p: [(p, oo.PROBE_FACE, k) for k in range(6)]
    first = oo.from_scene(og, mask, cams, probes, st, (640.0, 480.0))
    # the due probes' faces in pool order, then the enabled cameras; node 3 is disabled, 6 and 7 are not globally enabled
    assert keys(first) == faces(2) + faces(4) + faces(8) + [(1, oo.CAMERA, 0)]
    # Once probes were rendered: only the EachFrame probe comes back
    assert keys(oo.from_scene(og, mask, cams, probes, st, (640.0, 480.0))) == faces(4) + [(1, oo.CAMERA, 0)]
    # force_update (or a new record) makes a Once probe due for one call
    st.reset([8])
    assert keys(oo.from_scene(og, mask, cams, probes, st, (640.0, 480.0))) == faces(4) + faces(8) + [(1, oo.CAMERA, 0)]
    assert keys(oo.from_scene(og, mask, cams, probes, st, (640.0, 480.0))) == faces(4) + [(1, oo.CAMERA, 0)]
    # the probe translation is the global position plus rendering_position; faces never get an environment map
    o8 = [o for o in first if o["node"] == 8][0]
    assert np.array_equal(o8["translation"], og.global_transform(8)[12:15] + np.array((0.5, -1.0, 2.0), f32))
    assert all(o["environment_map"] == NONE for o in first if o["kind"] == oo.PROBE_FACE)


def test_render_target_frame_size_overrides_the_call():
    g = np.eye(4, dtype=f32).reshape(16)
    _, _, p_call = oo.camera_matrices(g, oo.Camera(), (100.0, 100.0))
    _, _, p_rt = oo.camera_matrices(g, oo.Camera(frame_size=(800.0, 200.0)), (100.0, 100.0))
    m22 = co.m22_of(1.2)
    assert p_call[0] == m22 and p_call[5] == m22
    assert p_rt[0] == m22 / f32(4.0) and p_rt[5] == m22


def test_projections_and_their_guards():
    fs = (300.0, 200.0)
    # z_near and z_far swapped: min / max restore them
    a = oo.projection(oo.PERSPECTIVE, 1.0, 0.5, 80.0, fs)
    b = oo.projection(oo.PERSPECTIVE, 1.0, 80.0, 0.5, fs)
    assert a.tobytes() == b.tobytes()
    # equal planes: z_far grows by 10 * f32::EPSILON
    c = oo.projection(oo.PERSPECTIVE, 1.0, 2.0, 2.0, fs)
    assert c.tobytes() == co.perspective(co.m22_of(1.0), f32(1.5), f32(2.0), f32(2.0) + co.LIMIT).tobytes()
    # orthographic: a vertical size below the limit is clamped, with its sign
    d = oo.projection(oo.ORTHOGRAPHIC, 0.0, 0.1, 10.0, fs)
    assert d[5] == f32(2.0) / (co.LIMIT + co.LIMIT)
    e = oo.projection(oo.ORTHOGRAPHIC, -1e-9, 0.1, 10.0, fs)
    assert e[5] == f32(2.0) / (-co.LIMIT - co.LIMIT)
    f = oo.projection(oo.ORTHOGRAPHIC, 5.0, 0.1, 10.0, fs)
    assert f[5] == f32(2.0) / f32(10.0) and f[0] == f32(2.0) / (f32(1.5) * f32(5.0) * f32(2.0))
    # a zero-height frame: the aspect is clamped to the limit, not inf or NaN
    with np.errstate(divide="ignore"):
        g = oo.projection(oo.PERSPECTIVE, 1.0, 0.5, 80.0, (300.0, 0.0))
    assert np.isfinite(g).all()


def test_scaled_rotated_camera_uses_its_columns_as_they_are():
    ang = f32(0.7)
    c, s = np.cos(ang, dtype=f32), np.sin(ang, dtype=f32)
    rot = np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]], f32)
    scl = np.diag(np.array([2.0, 3.0, 0.5], f32))
    m = np.eye(4, dtype=f32)
    m[:3, :3] = rot @ scl
    m[:3, 3] = (1.0, 2.0, -3.0)
    g = m.T.reshape(16).copy()  # column-major
    pos, view, _ = oo.camera_matrices(g, oo.Camera(), (640.0, 480.0))
    # look = column 2 (length 0.5), up = column 1 (length 3): not normalised before look_at_rh
    assert np.array_equal(view, ob.look_at_rh(g[12:15], g[12:15] + g[8:11], g[4:7]))
    assert not np.isclose(np.linalg.norm(g[8:11]), 1.0) and not np.isclose(np.linalg.norm(g[4:7]), 1.0)
    v = view.reshape(4, 4).T
    assert np.allclose(v[:3, :3] @ v[:3, :3].T, np.eye(3), atol=1e-6)
    assert np.allclose(v[:3, :3] @ pos + v[:3, 3], 0.0, atol=1e-5)
    assert np.allclose(-v[2, :3], g[8:11] / np.linalg.norm(g[8:11]), atol=1e-6)  # the camera looks along -z of its view


def test_probe_fov_is_the_point_lights_quarter_turn():
    """90f32.to_radians() = 90 * (PI / 180) in f32 equals FRAC_PI_2, so the probe faces share the point-light faces' m22."""
    rads_per_deg = f32(np.pi) / f32(180.0)
    assert f32(90.0) * rads_per_deg == so.FRAC_PI_2
    assert oo.FOV_90 == so.FRAC_PI_2
    assert co.m22_of(oo.FOV_90) == ob.perspective(1.0, float(so.FRAC_PI_2), 0.01, 10.0)[5]
    p = oo.projection(oo.PERSPECTIVE, oo.FOV_90, 0.1, 50.0, (1.0, 1.0))
    assert p.tobytes() == ob.perspective(1.0, float(so.FRAC_PI_2), 0.1, 50.0).tobytes()
