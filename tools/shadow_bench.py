#!/usr/bin/env python
"""Shadow-caster culls of one camera at scale: fyx_cull_shadow_casters (route a) against what a host does without it
(route b): fyx_cull_lights and the light list, the lights' global matrices read back, the shadow gating and light matrices
of renderer/light.rs:509-606, 695-763 rebuilt on the CPU, then fyx_cull with at most FYX_MAX_FRUSTA frusta per call and
every list read back.

Scene: 10 M nodes from scenegen (the node count of C4; no skinned units: the shadow cull reads node columns only) with
light nodes among them, in front of the camera.  Two loads: 8 spot + 8 point lights (56 maps) and 32 point lights
(192 maps).  The routes run in one process and alternate three times; both must give the same maps (light, face, cascade,
view_projection bits) and the same sets.  Each timed call starts from the camera cull (both routes need it, and route b's
culls replace it).  Prints one JSON line per load, with the card's name and power limit.

    python tools/shadow_bench.py [--nodes 10000000] [--steps 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import ctypes  # noqa: E402

import numpy as np  # noqa: E402

import fyrox_b200 as fb  # noqa: E402
from fyrox_b200 import camera  # noqa: E402
from fyrox_b200.scenegen import Scene  # noqa: E402

f32 = np.float32
_tanf = ctypes.CDLL("libm.so.6").tanf  # the platform's tanf, as the reference and fyx_set_light_sources
_tanf.restype, _tanf.argtypes = ctypes.c_float, [ctypes.c_float]
FRAC_PI_2 = f32(1.57079632679489661923)
EPS = f32(1.1920929e-07)
SETTINGS = (60.0, 60.0, 1, 1)  # spot / point shadows_distance, enabled
Z_NEAR = 0.01
NODE_BYTES = 4 + 4 + 24  # flags, render mask, world box: what one cull pass reads per node


# ---- route b: the host's restatement (light.rs, shadow/point.rs, nalgebra look_at_rh / new_perspective), f32 scalars ----
def dot3(u, v):
    return (f32(u[0]) * f32(v[0]) + f32(u[1]) * f32(v[1])) + f32(u[2]) * f32(v[2])


def cross3(u, v):
    return np.array([f32(u[1]) * f32(v[2]) - f32(u[2]) * f32(v[1]), f32(u[2]) * f32(v[0]) - f32(u[0]) * f32(v[2]),
                     f32(u[0]) * f32(v[1]) - f32(u[1]) * f32(v[0])], f32)


def look_at_rh(eye, target, up):
    fwd = np.array([target[k] - eye[k] for k in range(3)], f32)
    fl = np.sqrt(dot3(fwd, fwd))
    fwd = np.array([fwd[k] / fl for k in range(3)], f32)
    s = cross3(fwd, up)
    sl = np.sqrt(dot3(s, s))
    s = np.array([s[k] / sl for k in range(3)], f32)
    u = cross3(s, fwd)
    m = np.zeros(16, f32)
    m[0], m[4], m[8], m[12] = s[0], s[1], s[2], -dot3(s, eye)
    m[1], m[5], m[9], m[13] = u[0], u[1], u[2], -dot3(u, eye)
    m[2], m[6], m[10], m[14] = -fwd[0], -fwd[1], -fwd[2], dot3(fwd, eye)
    m[15] = 1.0
    return m


def perspective(m22, znear, zfar):
    m = np.zeros(16, f32)
    znear, zfar = f32(znear), f32(zfar)
    m[5] = m22
    m[0] = m22 / f32(1.0)
    m[10] = (zfar + znear) / (znear - zfar)
    m[14] = zfar * znear * f32(2.0) / (znear - zfar)
    m[11] = -1.0
    return m


def try_normalize(v, fallback):
    n = np.sqrt(dot3(v, v))
    return np.array(fallback, f32) if n <= EPS else np.array([v[k] / n for k in range(3)], f32)


def host_maps(ctx, cam_planes, cam_t, lights, sources):
    """Route b up to the culls: light list, matrices read back, gating, cascades, view_projection per map."""
    ctx.cull_lights()
    listed = ctx.get_visible_lights(0)
    rec = [n for n in listed.tolist() if n in sources]
    if not rec:
        return []
    g = ctx.get_global_matrices(np.array(rec, np.uint32))
    out = []
    for node, m in zip(rec, g):
        kind, cone, raw = sources[node]
        pos = m[12:15].astype(f32)
        d = pos - cam_t
        dist = np.sqrt(dot3(d, d))
        sd = f32(SETTINGS[0] if kind == fb.LIGHT_SPOT else SETTINGS[1])
        enabled = dist <= sd  # every light casts shadows; both kinds enabled
        radius = f32(1.0) * f32(raw)  # scenegen nodes carry no TRS record: unit scale
        inside = True
        for p in cam_planes:
            dd = dot3(p[:3], pos) + f32(p[3])
            if dd < -radius:
                inside = False
                break
            if abs(dd) < radius:
                break
        if not (enabled and inside):
            continue
        b1, b2 = sd * f32(0.2), sd * f32(0.4)
        e = cam_t - pos
        cascade = 0 if (dist < b1 or np.sqrt(dot3(e, e)) <= radius) else (1 if (dist > b1 and dist < b2) else 2)
        fovy = f32(cone) if kind == fb.LIGHT_SPOT else FRAC_PI_2
        proj = perspective(f32(1.0) / f32(_tanf(fovy / f32(2.0))), Z_NEAR, radius)
        if kind == fb.LIGHT_SPOT:
            emit = try_normalize(m[4:7], (0, 0, 1))
            up = try_normalize(m[8:11], (0, 1, 0))
            out.append((node, 0, cascade, fb.mat4_mul(proj, look_at_rh(pos, pos - emit, up))))
        else:
            for k, (look, up) in enumerate(camera.CUBE_FACES):
                out.append((node, k, cascade, fb.mat4_mul(proj, look_at_rh(pos, pos + np.array(look, f32), np.array(up, f32)))))
    return out


def route_b(ctx, cam_ff, cam_planes, cam_t, lights, sources, copy=True):
    ctx.cull([cam_ff])
    maps = host_maps(ctx, cam_planes, cam_t, lights, sources)
    lists = []
    for b in range(0, len(maps), 8):
        chunk = maps[b: b + 8]
        frusta = [fb.frustum_from_view_projection_matrix(m[3]) or fb.frustum_default() for m in chunk]
        ctx.cull(frusta, pass_flags=[fb.PASS_SHADOW] * len(frusta))
        lists += [ctx.get_visible(k, copy=copy) for k in range(len(chunk))]
    return maps, lists


def route_a(ctx, cam_ff, cam_t, copy=True):
    ctx.cull([cam_ff])
    ctx.cull_shadow_casters(0, cam_t, *SETTINGS)
    return ctx.get_shadow_maps(copy=copy)


def same(a, b):
    maps, entries = a
    bm, bl = b
    if len(maps) != len(bm):
        return False
    for m, (node, face, cascade, vp), lst in zip(maps, bm, bl):
        if (int(m["light"]), int(m["face"]), int(m["cascade"])) != (node, face, cascade) or m["view_projection"].tobytes() != vp.tobytes():
            return False
        if not np.array_equal(np.sort(entries[m["first"]: m["first"] + m["count"]]), np.sort(lst)):
            return False
    return True


def kernel_times(ctx, cam_ff, cam_t, sources, cam_planes, lights):
    """Per-kernel device time from a torch.profiler CUDA activity trace of one call of each route (a run of its own)."""
    try:
        import torch
        from torch.profiler import ProfilerActivity, profile
    except Exception as e:  # pragma: no cover
        return {"error": f"torch.profiler unavailable: {e}"}
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        route_a(ctx, cam_ff, cam_t)
        route_b(ctx, cam_ff, cam_planes, cam_t, lights, sources)
        torch.cuda.synchronize()
    us = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = getattr(ev, "cuda_time_total", 0.0)
        if t and ev.key.startswith(("void fyx::k_", "fyx::k_", "k_")):
            key = ev.key.split("(")[0].split("<")[0].split("::")[-1]
            us[key] = us.get(key, 0.0) + float(t)
    return us


def peak():
    p = os.path.join(REPO, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        return float(json.load(open(p))["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"
    return 3350.0, "H100 SXM data sheet: 3.35 TB/s HBM3 (not measured)"


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=10_000_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--radius", type=float, default=8.0)
    args = ap.parse_args()
    sc = Scene(args.nodes)
    ctx = fb.Context()
    flags = sc.flags.copy()
    ctx.set_topology(sc.parent, flags, sc.render_mask, sc.local_aabb, root=0)
    ctx.set_local_matrices(sc.local_m16)
    ctx.update_transforms(fb.UPDATE_ALL)
    cam_fo = camera.camera_frustum()
    planes, _ = fb.frustum_to_numpy(cam_fo)
    cam_t = np.zeros(3, f32)
    # light candidates: renderable nodes well inside the camera's view
    rng = np.random.default_rng(5)
    cand = rng.choice(np.flatnonzero(sc.flags & fb.NODE_RENDERABLE), 20000, replace=False).astype(np.uint32)
    pos = ctx.get_global_matrices(cand)[:, 12:15]
    gvis = fb.NODE_GLOBAL_VISIBILITY | fb.NODE_GLOBAL_ENABLED
    ok = ((ctx.get_global_flags(cand) & gvis) == gvis) & (pos[:, 2] < -8) & (pos[:, 2] > -50) & (np.abs(pos[:, 0]) < 0.3 * -pos[:, 2]) & (np.abs(pos[:, 1]) < 0.3 * -pos[:, 2])
    pool = np.sort(cand[ok])
    peak_gbs, peak_src = peak()
    gpu = card()
    for name, n_spot, n_point in (("8 spot + 8 point", 8, 8), ("32 point", 0, 32)):
        lights = np.sort(rng.choice(pool, n_spot + n_point, replace=False)).astype(np.uint32)
        kinds = np.array([fb.LIGHT_SPOT] * n_spot + [fb.LIGHT_POINT] * n_point)[rng.permutation(n_spot + n_point)]
        sources = {int(n): (int(k), float(f32(1.0)), float(f32(args.radius))) for n, k in zip(lights, kinds)}
        fl = flags.copy()
        fl[lights] |= fb.NODE_LIGHT | fb.NODE_CAST_SHADOWS
        ctx.set_flags(fl[lights], lights)
        ctx.update_transforms(fb.UPDATE_ALL)
        nodes = np.array(sorted(sources), np.uint32)
        rec = np.zeros(len(nodes), fb.Context.LIGHT_SOURCE_DTYPE)
        for k, n in enumerate(nodes.tolist()):
            rec[k] = sources[n]
        ctx.set_light_sources(rec, nodes)
        cam_ff = camera.camera_frustum()
        a = route_a(ctx, cam_ff, cam_t)
        b = route_b(ctx, cam_ff, planes, cam_t, lights, sources)
        identical = same(a, b)
        t = {"a": [], "b": []}
        # timed: both routes end with every list readable on the host (pinned library buffers, no numpy copies)
        for _ in range(3):  # alternate the routes three times
            for r in ("a", "b"):
                t0 = time.perf_counter()
                for _ in range(args.steps):
                    if r == "a":
                        route_a(ctx, cam_ff, cam_t, copy=False)
                    else:
                        route_b(ctx, cam_ff, planes, cam_t, lights, sources, copy=False)
                t[r].append((time.perf_counter() - t0) / args.steps * 1e3)
        a = route_a(ctx, cam_ff, cam_t)
        b = route_b(ctx, cam_ff, planes, cam_t, lights, sources)
        identical = identical and same(a, b)
        t0 = time.perf_counter()
        for _ in range(args.steps):
            ctx.cull([cam_ff])
            ctx.sync()
        cam_ms = (time.perf_counter() - t0) / args.steps * 1e3
        maps, entries = a
        n_maps = len(maps)
        kt = kernel_times(ctx, cam_ff, cam_t, sources, planes, lights)
        n = sc.capacity
        # algorithmic bytes per node: route a = count pass (node columns + one warp flag per 32 nodes) + emit pass over the
        # warps that have an entry; route b = one pass per 8 maps.  Lists: 4 B per entry in both.
        passes_b = (n_maps + 7) // 8
        cnt_us, emit_us, cull_us = kt.get("k_shadow_count", 0.0), kt.get("k_shadow_emit", 0.0), kt.get("k_cull", 0.0)
        out = {
            "tool": "shadow_bench", "load": name, "gpu": gpu, "nodes": n, "maps": n_maps, "entries": int(len(entries)),
            "identical": bool(identical),
            "ms_per_call_a": t["a"], "ms_per_call_b": t["b"], "ms_camera_cull_alone": cam_ms,
            "bytes_per_node_a": {"count_pass": NODE_BYTES + 4 / 32, "emit_pass_read_per_warp_with_entries": NODE_BYTES + 4 + 4 / 32},
            "bytes_per_node_b": {"per_pass": NODE_BYTES, "passes": passes_b, "total": NODE_BYTES * passes_b},
            "kernel_us": kt,
            "hbm_peak_gbs": peak_gbs, "hbm_peak_source": peak_src,
        }
        if cnt_us:
            out["k_shadow_count_GBps"] = NODE_BYTES * n / (cnt_us * 1e-6) / 1e9
            out["k_shadow_count_share_of_peak"] = out["k_shadow_count_GBps"] / peak_gbs
        if cull_us:
            out["k_cull_GBps_route_b"] = NODE_BYTES * n * (passes_b + 2) / (cull_us * 1e-6) / 1e9  # + the two camera culls
        out["k_shadow_emit_us"] = emit_us
        print(json.dumps(out), flush=True)
        ctx.set_light_sources(np.zeros(len(nodes), fb.Context.LIGHT_SOURCE_DTYPE), nodes)  # next load starts without records
        ctx.set_flags(flags[lights], lights)
    ctx.close()


if __name__ == "__main__":
    main()
