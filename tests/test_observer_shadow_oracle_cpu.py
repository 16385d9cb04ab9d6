"""The oracle of fyx_cull_scene_shadow_casters on its own (no GPU): every observer's shadow maps in render order, the
cascade camera each observer gives, the gates, and the premise of sharing spot and point maps between observers."""
import numpy as np
import pytest

import csm_oracle as co
import observer_oracle as oo
import observer_shadow_oracle as oso
import shadow_oracle as so
from test_gpu_observers import FRAME, ObserverScene

f32 = np.float32
SETTINGS = (40.0, 40.0, 1, 1)


def scene(seed, n=2500, n_cams=4, n_probes=3, pruners=True):
    s = ObserverScene(np.random.default_rng(seed), n, n_cams, n_probes, pruners=pruners)
    og = s.pr.oracle()
    obs = oo.from_scene(og, s.sc.mask, s.cams, s.probes, s.state, FRAME)
    return s, og, obs


def maps_of(s, og, o, **kw):
    sc = s.sc
    return oso.observer_maps(og, sc.flags, o, s.cams, FRAME, kw.pop("settings", SETTINGS), kw.pop("sources", sc.sources), sc.scale(), **kw)


def test_render_order_follows_each_light_list():
    s, og, obs = scene(5100)
    per = oso.scene_shadow_maps(og, s.sc.flags, obs, s.cams, FRAME, SETTINGS, s.sc.sources, s.sc.scale())
    assert sum(len(m) for m in per) > 20
    for o, maps in zip(obs, per):
        order = {int(x): k for k, x in enumerate(o["lights"])}
        lights = [m["light"] for m in maps]
        assert all(x in order for x in lights) and [order[x] for x in lights] == sorted(order[x] for x in lights)
        k = 0
        while k < len(maps):  # each light's maps together: cube faces 0..5, cascades 0..2, one spot map
            light = maps[k]["light"]
            run = [m for m in maps[k:] if m["light"] == light][: {so.LIGHT_SPOT: 1, so.LIGHT_POINT: 6, so.LIGHT_DIRECTIONAL: 3}[s.sc.sources[light][0]]]
            if s.sc.sources[light][0] == so.LIGHT_POINT:
                assert [m["face"] for m in run] == list(range(6))
            if s.sc.sources[light][0] == so.LIGHT_DIRECTIONAL:
                assert [m["cascade"] for m in run] == [0, 1, 2]
            assert all(m["mask"] == int(o["render_mask"]) for m in run)
            k += len(run)


def test_probe_faces_take_any_square_frame():
    s, og, obs = scene(5200)
    faces = [o for o in obs if o["kind"] == oo.PROBE_FACE]
    assert faces
    got_dir = False
    for o in faces[:6]:
        a = maps_of(s, og, o)
        for size in (1.0, 256.0, 777.0):
            b = maps_of(s, og, o, probe_frame=(size, size))
            assert [m["view_projection"].tobytes() for m in a] == [m["view_projection"].tobytes() for m in b]
        got_dir |= any(s.sc.sources[m["light"]][0] == so.LIGHT_DIRECTIONAL for m in a)
    # a frame that is not square moves the cascades: the aspect, not the size, is what a face's projection takes
    o = next(o for o in faces if any(s.sc.sources[m["light"]][0] == so.LIGHT_DIRECTIONAL for m in maps_of(s, og, o)))
    a = [m for m in maps_of(s, og, o) if m["cascade"] and s.sc.sources[m["light"]][0] == so.LIGHT_DIRECTIONAL]
    b = [m for m in maps_of(s, og, o, probe_frame=(1280.0, 720.0)) if m["cascade"] and s.sc.sources[m["light"]][0] == so.LIGHT_DIRECTIONAL]
    assert got_dir and [m["view_projection"].tobytes() for m in a] != [m["view_projection"].tobytes() for m in b]


def test_render_target_camera_uses_its_own_frame_size():
    s, og, obs = scene(5300, n_cams=6)
    cams = [o for o in obs if o["kind"] == oo.CAMERA and s.cams[o["node"]].frame_size != (0.0, 0.0)]
    assert cams
    o = cams[0]
    own = oso.csm_camera(o, s.cams, FRAME)
    assert own.frame_size == (640.0, 640.0)
    call = oso.csm_camera(o, {o["node"]: oo.Camera(**{**s.cams[o["node"]].__dict__, "frame_size": (0.0, 0.0)})}, FRAME)
    assert call.frame_size == FRAME
    sl_own = co.slice_corners(own, *co.cascade_depths(own, co.CSM_DEFAULT, 1))
    sl_call = co.slice_corners(call, *co.cascade_depths(call, co.CSM_DEFAULT, 1))
    assert not np.array_equal(sl_own, sl_call)


def test_a_light_in_one_face_list_and_not_another():
    s, og, obs = scene(5400, n_probes=4)
    split = False
    for p in {o["node"] for o in obs if o["kind"] == oo.PROBE_FACE}:
        faces = [o for o in obs if o["node"] == p and o["kind"] == oo.PROBE_FACE]
        per = [maps_of(s, og, o) for o in faces]
        for o, maps in zip(faces, per):
            assert {m["light"] for m in maps} <= {int(x) for x in o["lights"]}
        sets = [{m["light"] for m in maps} for maps in per]
        split |= any(a != b for a in sets for b in sets)
        # the six faces of a probe share one translation: a light's cascade index is the same in each
        casc = {}
        for maps in per:
            for m in maps:
                if s.sc.sources[m["light"]][0] != so.LIGHT_DIRECTIONAL:
                    casc.setdefault(m["light"], set()).add(m["cascade"])
        assert all(len(v) == 1 for v in casc.values())
    assert split


def test_lights_without_a_record_and_csm_disabled():
    s, og, obs = scene(5200)
    o = max(obs, key=lambda o: len(maps_of(s, og, o)))
    full = maps_of(s, og, o)
    gone = full[0]["light"]
    rest = maps_of(s, og, o, sources={k: v for k, v in s.sc.sources.items() if k != gone})
    assert gone not in {m["light"] for m in rest}
    assert [(m["light"], m["face"], m["cascade"]) for m in rest] == [(m["light"], m["face"], m["cascade"]) for m in full if m["light"] != gone]
    dirs = [m for o2 in obs for m in maps_of(s, og, o2) if s.sc.sources[m["light"]][0] == so.LIGHT_DIRECTIONAL]
    assert dirs
    for o2 in obs:
        off = maps_of(s, og, o2, csm_enabled=False)
        assert not any(s.sc.sources[m["light"]][0] == so.LIGHT_DIRECTIONAL for m in off)
        assert [(m["light"], m["face"]) for m in off] == [(m["light"], m["face"]) for m in maps_of(s, og, o2)
                                                           if s.sc.sources[m["light"]][0] != so.LIGHT_DIRECTIONAL]


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_equal_keys_give_equal_maps(seed):
    """The premise of sharing: spot and point maps with equal (light, face, cascade, mask) are the same map for every
    observer — view_projection, LOD observer and list — on scenes with LOD ranges and static batches."""
    s, og, obs = scene(5600 + seed, n_cams=5, n_probes=3)
    rows, shared = {}, 0
    for o in obs:
        for m in maps_of(s, og, o):
            if s.sc.sources[m["light"]][0] == so.LIGHT_DIRECTIONAL:
                continue
            key = (m["light"], m["face"], m["cascade"], m["mask"])
            val = (m["view_projection"].tobytes(), np.asarray(m["observer"][0], f32).tobytes(), f32(m["observer"][1]).tobytes(),
                   f32(m["observer"][2]).tobytes(), m["visible"].tobytes())
            if key in rows:
                assert rows[key] == val, key
                shared += 1
            rows[key] = val
    assert shared > 0 and s.pr.ranges
