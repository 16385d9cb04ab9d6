#!/usr/bin/env python
"""The shadow maps of every scene observer at scale: 2 cameras and 4 reflection probes updated every frame (26 observers),
8 spot, 8 point and 1 directional light with records.

    (a) fyx_cull_scene_observers + fyx_cull_scene_shadow_casters + fyx_pack_shadow_instances: one map table for all
        observers, spot and point maps that several observers render culled once, one node pass;
    (b) fyx_cull_scene_observers, then what a host does without (a), per observer: fyx_cull on its frustum and mask,
        fyx_cull_lights, fyx_cull_shadow_casters_pruned with a csm camera built from its record, and one
        fyx_pack_shadow_instances.  The observer table is read back once (a host needs it to build the csm cameras).
Both routes leave the lists and instances on the device while they are timed.

Scene: 10 M scenegen nodes, with and without LOD ranges (about 1 % of the nodes) and static batches (about 0.1 %).  The
routes alternate three times in one process, each call timed on the host clock around work that ends in a synchronise; (a)
and (b) must give the same maps and sets.  A separate torch.profiler run gives the count- and emit-pass kernel times.
Prints one JSON line per scene, with the card's name and power limit read in the same run.

    python tools/scene_shadow_bench.py [--nodes 10000000] [--steps 3] [--profile-dir DIR]
"""
import argparse
import json
import os
import re
import subprocess
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import numpy as np  # noqa: E402

import fyrox_b200 as fb  # noqa: E402
from fyrox_b200.scenegen import Scene  # noqa: E402

f32 = np.float32
LEVELS = [(0.0, 0.3), (0.3, 0.8), (0.8, 4.0)]
FRAME = np.array([1920.0, 1080.0], f32)
SETTINGS = (60.0, 60.0, 1, 1)  # spot / point shadows_distance, enabled
CAM = (1, fb.PROJECTION_PERSPECTIVE, 1.2, 0.1, 200.0, (0.0, 0.0))
FOV_90 = float(f32(np.pi / 2))


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:
        return f"unknown ({e})"


def route_a(ctx):
    ctx.cull_scene_observers(FRAME)
    ctx.cull_scene_shadow_casters(*SETTINGS)
    ctx.pack_shadow_instances()


def csm_camera(r):
    if int(r["kind"]) == fb.OBSERVER_CAMERA:
        return fb.Context.csm_camera(r["view"], FRAME, float(r["z_near"]), float(r["z_far"]), fov=CAM[2])
    return fb.Context.csm_camera(r["view"], (1.0, 1.0), float(r["z_near"]), float(r["z_far"]), fov=FOV_90)


def route_b(ctx, read=False):
    ctx.cull_scene_observers(FRAME)
    table, _, _ = ctx.get_scene_observers()
    out = []
    for r in table:
        ctx.cull([fb.frustum_from_view_projection_matrix(r["view_projection"]) or fb.frustum_default()], cam_mask=[int(r["render_mask"])])
        ctx.cull_lights()
        ctx.cull_shadow_casters(0, r["translation"], *SETTINGS, csm_camera=csm_camera(r), prune=True)
        ctx.pack_shadow_instances()
        if read:
            out.append(maps_of(ctx))
    return out


def maps_of(ctx):
    maps, entries = ctx.get_shadow_maps()
    return [(int(m["light"]), int(m["face"]), int(m["cascade"]), m["view_projection"].tobytes(),
             np.sort(entries[m["first"]: m["first"] + m["count"]]).tobytes()) for m in maps]


def read_a(ctx):
    ctx.cull_scene_observers(FRAME)
    table, _, _ = ctx.get_scene_observers()
    ctx.cull_scene_shadow_casters(*SETTINGS)
    rows = maps_of(ctx)
    refs = ctx.get_scene_shadow_maps()
    out = [[] for _ in range(len(table))]
    for r in refs:
        out[int(r["observer"])].append(rows[int(r["map"])])
    return out, len(refs), len(rows), int(ctx.get_shadow_maps()[1].size)


def profile(ctx, out_dir, tag):
    import torch
    from torch.profiler import ProfilerActivity, profile as prof

    with prof(activities=[ProfilerActivity.CUDA]) as p:
        for _ in range(3):
            route_a(ctx)
    times = {}
    # this call's kernels: its table kernel, the node passes in its form (kFormSceneShadow = 2, their last template argument;
    # the observer call runs them in another form) and the scan
    passes = re.compile(r"k_shadow_(pruners|count|emit)<.*\b2>")
    for e in p.key_averages():
        if "k_scene_shadow" in e.key or "k_shadow_scan" in e.key or passes.search(e.key):
            times[e.key] = round(e.device_time_total / max(e.count, 1) / 1e3, 4)  # ms per launch
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        p.export_chrome_trace(os.path.join(out_dir, f"scene_shadow_{tag}.json"))
    return times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=10_000_000)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--profile-dir", default=None)
    args = ap.parse_args()
    gpu = card()
    sc = Scene(args.nodes)
    n = sc.capacity
    rng = np.random.default_rng(12)
    alive = np.flatnonzero(sc.flags & fb.NODE_ALIVE)
    alive = alive[alive > 0]
    n_children = np.bincount(sc.parent[sc.parent != 0xFFFFFFFF].astype(np.int64), minlength=n)
    parents = alive[n_children[alive] > 0]
    batches = np.sort(rng.choice(parents, min(parents.size, max(1, n // 1000)), replace=False)).astype(np.uint32)
    lod_nodes = np.sort(rng.choice(alive, max(1, n // 100), replace=False)).astype(np.uint32)
    ranges = np.array([LEVELS[k] for k in rng.integers(0, len(LEVELS), lod_nodes.size)], f32)
    pool = np.setdiff1d(alive, np.concatenate([batches, lod_nodes]))
    obs_nodes = np.sort(rng.choice(pool, 6, replace=False)).astype(np.uint32)
    cams, probes = obs_nodes[:2], obs_nodes[2:]
    lights = np.sort(rng.choice(np.setdiff1d(pool, obs_nodes), 17, replace=False)).astype(np.uint32)
    kinds = [fb.LIGHT_SPOT] * 8 + [fb.LIGHT_POINT] * 8 + [fb.LIGHT_DIRECTIONAL]
    rng.shuffle(kinds)
    src = np.zeros(len(lights), fb.Context.LIGHT_SOURCE_DTYPE)
    src[:] = [(k, 1.0, 15.0) for k in kinds]
    base = sc.flags.copy()
    base[batches] |= fb.NODE_RENDERABLE
    base[lights] |= fb.NODE_LIGHT | fb.NODE_CAST_SHADOWS
    base[probes] |= fb.NODE_REFLECTION_PROBE
    for name, pruned in (("no LOD ranges or static batches", False), ("LOD ranges and static batches", True)):
        flags = base.copy()
        if pruned:
            flags[batches] |= fb.NODE_STATIC_BATCH
        ctx = fb.Context()
        ctx.enable_instances(True)
        ctx.set_topology(sc.parent, flags, sc.render_mask, sc.local_aabb, root=0)
        ctx.set_local_matrices(sc.local_m16)
        ctx.update_transforms(fb.UPDATE_ALL)
        if pruned:
            ctx.set_lod_ranges(ranges, lod_nodes)
        cam = np.zeros(2, fb.Context.CAMERA_DTYPE)
        cam[:] = CAM
        ctx.set_cameras(cams, cam)
        pr = np.zeros(4, fb.Context.PROBE_DTYPE)
        pr[:] = (1, fb.PROBE_UPDATE_EACH_FRAME, 0.1, 60.0, (0.0, 0.0, 0.0))
        ctx.set_reflection_probes(probes, pr)
        ctx.set_light_sources(src, lights)
        a, n_refs, n_maps, n_entries = read_a(ctx)
        identical = a == route_b(ctx, read=True)
        t = {"a": [], "b": []}
        for _ in range(3):  # alternate the routes three times
            for r in ("a", "b"):
                t0 = time.perf_counter()
                for _ in range(args.steps):
                    route_a(ctx) if r == "a" else route_b(ctx)
                ctx.sync()
                t[r].append((time.perf_counter() - t0) / args.steps * 1e3)
        a2, _, _, _ = read_a(ctx)
        identical = identical and a2 == route_b(ctx, read=True)
        kernels = profile(ctx, args.profile_dir, "pruned" if pruned else "plain")
        print(json.dumps({
            "tool": "scene_shadow_bench", "scene": name, "gpu": gpu, "nodes": n, "observers": len(a), "referenced_maps": n_refs,
            "distinct_maps": n_maps, "entries": n_entries, "lod_objects": int(lod_nodes.size) if pruned else 0,
            "static_batches": int(batches.size) if pruned else 0, "identical_a_b": bool(identical),
            "ms_per_call_a_device": [round(x, 3) for x in t["a"]], "ms_per_call_b_host_route": [round(x, 3) for x in t["b"]],
            "kernel_ms_per_launch": kernels,
        }), flush=True)
        ctx.close()


if __name__ == "__main__":
    main()
