#!/usr/bin/env python
"""Cascaded shadow maps at scale: fyx_cull_shadow_casters_csm + fyx_pack_shadow_instances (route a) against what a host
does without them (route b): the light list and the lights' global matrices read back, the spot and point maps rebuilt on
the CPU (tools/shadow_bench.py), each directional light's three cascades rebuilt on the CPU (CsmRenderer::render,
renderer/shadow/csm.rs:165-249, through the f32 restatement of tests/csm_oracle.py), then per 8 maps fyx_cull with
FYX_PASS_SHADOW and one fyx_pack_instances per map.

Scene: 10 M scenegen nodes, every node in one of 64 bundles, light nodes in front of the camera.  Loads: 1 sun, 4 suns,
and 1 sun + 8 spot + 8 point lights.  The camera: perspective, 60° fov, z 0.1 .. 150, a 1920 x 1080 frame, default split
options (Absolute 5 / 25 / 64).  Both routes start from the camera cull and end with every map's instances in device
memory.  They run in one process and alternate three times; maps (light, face, cascade, view_projection bits), sets and
packed instances must be identical.  Prints one JSON line per load with the card's name and power limit and per-kernel
device times from torch.profiler.

    python tools/csm_bench.py [--nodes 10000000] [--steps 3]
"""
import argparse
import json
import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tests"))
import numpy as np  # noqa: E402

import csm_oracle as co  # noqa: E402
import shadow_bench as sb  # noqa: E402
import shadow_instances_bench as sib  # noqa: E402

import fyrox_b200 as fb  # noqa: E402
from fyrox_b200 import camera  # noqa: E402
from fyrox_b200.scenegen import Scene  # noqa: E402

f32 = np.float32
FOV = float(np.deg2rad(60.0))
FRAME = (1920.0, 1080.0)
Z_NEAR, Z_FAR = 0.1, 150.0


def host_maps(ctx, planes, cam_t, lights, sources, oc):
    """Route b up to the culls: [(light, face, cascade, view_projection, view)] in the light loop's order."""
    sp = {n: s for n, s in sources.items() if s[0] != fb.LIGHT_DIRECTIONAL}
    ctx.cull_lights()  # (shadow_bench.host_maps culls the lights again for its own list)
    other = sb.host_maps(ctx, planes, cam_t, lights, sp) if sp else []
    views = sib.views_of(ctx, other)
    by_light = {}
    for m, v in zip(other, views):
        by_light.setdefault(m[0], []).append(m + (v,))
    listed = ctx.get_visible_lights(0).tolist()
    suns = [n for n in listed if sources.get(n, (0,))[0] == fb.LIGHT_DIRECTIONAL]
    g = dict(zip(suns, ctx.get_global_matrices(np.array(suns, np.uint32)))) if suns else {}
    out = []
    for n in listed:
        if n in g:  # cast_shadows, csm enabled, unit scale: radius f32::MAX always meets the camera frustum
            with np.errstate(all="ignore"):
                for i, (v, vp) in enumerate(co.cascades(oc, co.CSM_DEFAULT, g[n][4:7].astype(f32), g[n][8:11].astype(f32))):
                    out.append((n, 0, i, vp, v))
        else:
            out += by_light.get(n, [])
    return out


def route_a(ctx, cam_ff, cam_t, fc):
    ctx.cull([cam_ff])
    ctx.cull_shadow_casters(0, cam_t, *sb.SETTINGS, csm_camera=fc)
    ctx.pack_shadow_instances()


def route_b(ctx, cam_ff, planes, cam_t, lights, sources, oc, read=False):
    ctx.cull([cam_ff])
    maps = host_maps(ctx, planes, cam_t, lights, sources, oc)
    got = []
    for b in range(0, len(maps), 8):
        chunk = maps[b: b + 8]
        frusta = [fb.frustum_from_view_projection_matrix(m[3]) or fb.frustum_default() for m in chunk]
        ctx.cull(frusta, pass_flags=[fb.PASS_SHADOW] * len(frusta))
        for k, m in enumerate(chunk):
            if read:
                got.append((m, np.sort(ctx.get_visible(k)), sib.canon(ctx.pack_instances(k, m[4], m[3]))))
            else:
                ctx._chk(ctx._lib.fyx_pack_instances(ctx._h, k, m[4].ctypes.data, m[3].ctypes.data))
    return got


def identical(ctx, cam_ff, planes, cam_t, lights, sources, oc, fc):
    route_a(ctx, cam_ff, cam_t, fc)
    maps, entries = ctx.get_shadow_maps()
    a = [(int(m["light"]), int(m["face"]), int(m["cascade"]), m["view_projection"].tobytes(), np.sort(entries[m["first"]: m["first"] + m["count"]]).tobytes(),
          sib.canon(ctx.get_shadow_instances(k))) for k, m in enumerate(maps)]
    b = [(m[0], m[1], m[2], m[3].tobytes(), vis.tobytes(), inst) for m, vis, inst in route_b(ctx, cam_ff, planes, cam_t, lights, sources, oc, read=True)]
    n_inst = sum(len(x[5][1]) // 4 for x in a)
    return a == b, len(maps), sum(1 for x in a if sources[x[0]][0] == fb.LIGHT_DIRECTIONAL), int(len(entries)), n_inst


def kernel_times(ctx, fn):
    import torch
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    us = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = getattr(ev, "cuda_time_total", 0.0)
        name = sib.re.search(r"\b(k_\w+)", ev.key)
        if t and name:
            us[name.group(1)] = us.get(name.group(1), 0.0) + float(t)
    return us


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=10_000_000)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--radius", type=float, default=8.0)
    ap.add_argument("--bundles", type=int, default=64)
    args = ap.parse_args()
    sc = Scene(args.nodes)
    ctx = fb.Context()
    flags = sc.flags.copy()
    ctx.set_topology(sc.parent, flags, sc.render_mask, sc.local_aabb, root=0)
    ctx.set_local_matrices(sc.local_m16)
    ctx.update_transforms(fb.UPDATE_ALL)
    rng = np.random.default_rng(5)
    ctx.set_bundle_ids(rng.integers(0, args.bundles, sc.capacity).astype(np.uint32))
    ctx.enable_instances()
    cam_fo = camera.camera_frustum()
    planes, _ = fb.frustum_to_numpy(cam_fo)
    cam_t = np.zeros(3, f32)
    view = sb.look_at_rh(np.zeros(3, f32), np.array([0, 0, -1], f32), np.array([0, 1, 0], f32))
    oc = co.CsmCamera(co.PERSPECTIVE, FOV, Z_NEAR, Z_FAR, FRAME, view)
    fc = fb.Context.csm_camera(view, FRAME, Z_NEAR, Z_FAR, fov=FOV)
    cand = rng.choice(np.flatnonzero(sc.flags & fb.NODE_RENDERABLE), 20000, replace=False).astype(np.uint32)
    pos = ctx.get_global_matrices(cand)[:, 12:15]
    gvis = fb.NODE_GLOBAL_VISIBILITY | fb.NODE_GLOBAL_ENABLED
    ok = ((ctx.get_global_flags(cand) & gvis) == gvis) & (pos[:, 2] < -8) & (pos[:, 2] > -50) & (np.abs(pos[:, 0]) < 0.3 * -pos[:, 2]) & (np.abs(pos[:, 1]) < 0.3 * -pos[:, 2])
    pool = np.sort(cand[ok])
    gpu = sb.card()
    for name, n_sun, n_spot, n_point in (("1 sun", 1, 0, 0), ("4 suns", 4, 0, 0), ("1 sun + 8 spot + 8 point", 1, 8, 8)):
        n = n_sun + n_spot + n_point
        lights = np.sort(rng.choice(pool, n, replace=False)).astype(np.uint32)
        kinds = np.array([fb.LIGHT_DIRECTIONAL] * n_sun + [fb.LIGHT_SPOT] * n_spot + [fb.LIGHT_POINT] * n_point)[rng.permutation(n)]
        sources = {int(nd): (int(k), float(f32(1.0)), float(f32(args.radius))) for nd, k in zip(lights, kinds)}
        sib.maps_kind.clear()
        sib.maps_kind.update({nd: k for nd, (k, _, _) in sources.items()})
        fl = flags.copy()
        fl[lights] |= fb.NODE_LIGHT | fb.NODE_CAST_SHADOWS
        ctx.set_flags(fl[lights], lights)
        ctx.update_transforms(fb.UPDATE_ALL)
        nodes = np.array(sorted(sources), np.uint32)
        rec = np.zeros(len(nodes), fb.Context.LIGHT_SOURCE_DTYPE)
        for k, nd in enumerate(nodes.tolist()):
            rec[k] = sources[nd]
        ctx.set_light_sources(rec, nodes)
        cam_ff = camera.camera_frustum()
        same, n_maps, n_casc, n_entries, n_inst = identical(ctx, cam_ff, planes, cam_t, lights, sources, oc, fc)
        t = {"a": [], "b": []}
        for _ in range(3):  # alternate the routes three times
            for r in ("a", "b"):
                t0 = time.perf_counter()
                for _ in range(args.steps):
                    if r == "a":
                        route_a(ctx, cam_ff, cam_t, fc)
                    else:
                        route_b(ctx, cam_ff, planes, cam_t, lights, sources, oc)
                ctx.sync()
                t[r].append((time.perf_counter() - t0) / args.steps * 1e3)
        same2 = identical(ctx, cam_ff, planes, cam_t, lights, sources, oc, fc)[0]
        ka = kernel_times(ctx, lambda: route_a(ctx, cam_ff, cam_t, fc))
        kb = kernel_times(ctx, lambda: route_b(ctx, cam_ff, planes, cam_t, lights, sources, oc))
        out = {
            "tool": "csm_bench", "load": name, "gpu": gpu, "nodes": sc.capacity, "maps": n_maps, "cascade_maps": n_casc, "entries": n_entries,
            "instances": n_inst, "identical": bool(same and same2),
            "ms_per_call_a": t["a"], "ms_per_call_b": t["b"],
            "device_us_a": sum(ka.values()), "device_us_b": sum(kb.values()),
            "k_shadow_frusta_us": ka.get("k_shadow_frusta", 0.0), "k_shadow_count_us": ka.get("k_shadow_count", 0.0),
            "k_shadow_emit_us": ka.get("k_shadow_emit", 0.0), "kernel_us_a": ka, "kernel_us_b": kb,
        }
        print(json.dumps(out), flush=True)
        ctx.set_light_sources(np.zeros(len(nodes), fb.Context.LIGHT_SOURCE_DTYPE), nodes)
        ctx.set_flags(flags[lights], lights)
    ctx.close()


if __name__ == "__main__":
    main()
