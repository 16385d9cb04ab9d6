#!/usr/bin/env python
"""The shadow maps' instances at scale: fyx_cull_shadow_casters + fyx_pack_shadow_instances (route a) against what a host
does without them (route b): the maps rebuilt on the CPU (tools/shadow_bench.py), then per 8 maps fyx_cull and one
fyx_pack_instances per map.

Scene and loads as tools/shadow_bench.py: 10 M scenegen nodes, 8 spot + 8 point lights (56 maps) and 32 point lights
(192 maps), every node in one of 64 bundles.  Both routes end with every map's instances in device memory.  They run in
one process and alternate three times; their packed instances must be identical per map (bundle tables bit for bit,
instances per (node, surface): the order inside a bundle is unspecified).  Prints one JSON line per load with the card's
name and power limit, per-kernel times from torch.profiler and the scatter kernel's algorithmic rate.

    python tools/shadow_instances_bench.py [--nodes 10000000] [--steps 3]
"""
import argparse
import json
import os
import re
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np  # noqa: E402

import shadow_bench as sb  # noqa: E402

import fyrox_b200 as fb  # noqa: E402
from fyrox_b200 import camera  # noqa: E402
from fyrox_b200.scenegen import Scene  # noqa: E402

f32 = np.float32
# k_shadow_inst_scatter per instance (single-surface nodes): reads entry slot + node 8, sort index 8, bundle id 4, skinning
# surface 4, flags 4, bin offset + cursor 8, global rows 48; writes node 4, sort index 8, surface 4, skin 4, matrices 128
SCATTER_BYTES = 8 + 8 + 4 + 4 + 4 + 8 + 48 + 4 + 8 + 4 + 4 + 128


def views_of(ctx, maps):
    """The view matrix of each host-built map (shadow_bench.host_maps), as light.rs / shadow/point.rs build it."""
    out = []
    g = ctx.get_global_matrices(np.array([m[0] for m in maps], np.uint32)) if maps else []
    for (node, face, _, vp), m in zip(maps, g):
        pos = m[12:15].astype(f32)
        if maps_kind[node] == fb.LIGHT_SPOT:
            emit = sb.try_normalize(m[4:7], (0, 0, 1))
            up = sb.try_normalize(m[8:11], (0, 1, 0))
            out.append(sb.look_at_rh(pos, pos - emit, up))
        else:
            look, up = camera.CUBE_FACES[face]
            out.append(sb.look_at_rh(pos, pos + np.array(look, f32), np.array(up, f32)))
    return out


maps_kind = {}


def route_a(ctx, cam_ff, cam_t):
    ctx.cull([cam_ff])
    ctx.cull_shadow_casters(0, cam_t, *sb.SETTINGS)
    ctx.pack_shadow_instances()


def route_b(ctx, cam_ff, planes, cam_t, lights, sources):
    ctx.cull([cam_ff])
    maps = sb.host_maps(ctx, planes, cam_t, lights, sources)
    views = views_of(ctx, maps)
    packed = []
    for b in range(0, len(maps), 8):
        chunk = maps[b: b + 8]
        frusta = [fb.frustum_from_view_projection_matrix(m[3]) or fb.frustum_default() for m in chunk]
        ctx.cull(frusta, pass_flags=[fb.PASS_SHADOW] * len(frusta))
        for k, m in enumerate(chunk):
            ctx._chk(ctx._lib.fyx_pack_instances(ctx._h, k, views[b + k].ctypes.data, m[3].ctypes.data))
            packed.append((b, k, views[b + k], m[3]))
    return packed


def canon(inst):
    o = np.lexsort((inst["surface"], inst["node"]))
    return (inst["bundles"].tobytes(),) + tuple(inst[k][o].tobytes() for k in ("node", "surface", "sort_index", "world", "wvp"))


def identical(ctx, cam_ff, planes, cam_t, lights, sources):
    route_a(ctx, cam_ff, cam_t)
    n_maps = len(ctx.get_shadow_maps()[0])
    a = [canon(ctx.get_shadow_instances(m)) for m in range(n_maps)]
    ctx.cull([cam_ff])
    maps = sb.host_maps(ctx, planes, cam_t, lights, sources)
    views = views_of(ctx, maps)
    b = []
    for s in range(0, len(maps), 8):
        chunk = maps[s: s + 8]
        frusta = [fb.frustum_from_view_projection_matrix(m[3]) or fb.frustum_default() for m in chunk]
        ctx.cull(frusta, pass_flags=[fb.PASS_SHADOW] * len(frusta))
        b += [canon(ctx.pack_instances(k, views[s + k], m[3])) for k, m in enumerate(chunk)]
    n_inst = sum(len(x[1]) // 4 for x in a)
    return a == b and len(a) == len(maps), n_maps, n_inst


def kernel_times(ctx, cam_ff, planes, cam_t, lights, sources):
    import torch
    from torch.profiler import ProfilerActivity, profile

    out = {}
    for name, fn in (("a", lambda: route_a(ctx, cam_ff, cam_t)), ("b", lambda: route_b(ctx, cam_ff, planes, cam_t, lights, sources))):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        us = {}
        for ev in prof.key_averages():
            t = getattr(ev, "device_time_total", None)
            if t is None:
                t = getattr(ev, "cuda_time_total", 0.0)
            name_ = re.search(r"\b(k_\w+)", ev.key)
            if t and name_:
                us[name_.group(1)] = us.get(name_.group(1), 0.0) + float(t)
        out[name] = us
    return out


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
    cand = rng.choice(np.flatnonzero(sc.flags & fb.NODE_RENDERABLE), 20000, replace=False).astype(np.uint32)
    pos = ctx.get_global_matrices(cand)[:, 12:15]
    gvis = fb.NODE_GLOBAL_VISIBILITY | fb.NODE_GLOBAL_ENABLED
    ok = ((ctx.get_global_flags(cand) & gvis) == gvis) & (pos[:, 2] < -8) & (pos[:, 2] > -50) & (np.abs(pos[:, 0]) < 0.3 * -pos[:, 2]) & (np.abs(pos[:, 1]) < 0.3 * -pos[:, 2])
    pool = np.sort(cand[ok])
    peak_gbs, peak_src = sb.peak()
    gpu = sb.card()
    for name, n_spot, n_point in (("8 spot + 8 point", 8, 8), ("32 point", 0, 32)):
        lights = np.sort(rng.choice(pool, n_spot + n_point, replace=False)).astype(np.uint32)
        kinds = np.array([fb.LIGHT_SPOT] * n_spot + [fb.LIGHT_POINT] * n_point)[rng.permutation(n_spot + n_point)]
        sources = {int(n): (int(k), float(f32(1.0)), float(f32(args.radius))) for n, k in zip(lights, kinds)}
        maps_kind.clear()
        maps_kind.update({n: k for n, (k, _, _) in sources.items()})
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
        same, n_maps, n_inst = identical(ctx, cam_ff, planes, cam_t, lights, sources)
        t = {"a": [], "b": []}
        for _ in range(3):  # alternate the routes three times
            for r in ("a", "b"):
                t0 = time.perf_counter()
                for _ in range(args.steps):
                    if r == "a":
                        route_a(ctx, cam_ff, cam_t)
                    else:
                        route_b(ctx, cam_ff, planes, cam_t, lights, sources)
                ctx.sync()
                t[r].append((time.perf_counter() - t0) / args.steps * 1e3)
        same2, _, _ = identical(ctx, cam_ff, planes, cam_t, lights, sources)
        kt = kernel_times(ctx, cam_ff, planes, cam_t, lights, sources)
        sc_us = kt["a"].get("k_shadow_inst_scatter", 0.0)
        pack_a = sum(v for k, v in kt["a"].items() if k in ("k_shadow_inst_keys", "k_bin_reduce", "k_bin_scan", "k_bin_downsweep", "k_shadow_inst_scatter"))
        pack_b = sum(v for k, v in kt["b"].items() if k in ("k_inst_keys", "k_inst_scan", "k_inst_scatter"))
        out = {
            "tool": "shadow_instances_bench", "load": name, "gpu": gpu, "nodes": sc.capacity, "maps": n_maps, "instances": n_inst,
            "bundle_ids": args.bundles, "identical": bool(same and same2),
            "ms_per_call_a": t["a"], "ms_per_call_b": t["b"],
            "pack_kernels_us_a": pack_a, "pack_kernels_us_b": pack_b, "kernel_us": kt,
            "scatter_bytes_per_instance": SCATTER_BYTES, "hbm_peak_gbs": peak_gbs, "hbm_peak_source": peak_src,
        }
        if sc_us:
            out["k_shadow_inst_scatter_GBps"] = SCATTER_BYTES * n_inst / (sc_us * 1e-6) / 1e9
            out["k_shadow_inst_scatter_share_of_peak"] = out["k_shadow_inst_scatter_GBps"] / peak_gbs
        print(json.dumps(out), flush=True)
        ctx.set_light_sources(np.zeros(len(nodes), fb.Context.LIGHT_SOURCE_DTYPE), nodes)
        ctx.set_flags(flags[lights], lights)
    ctx.close()


if __name__ == "__main__":
    main()
