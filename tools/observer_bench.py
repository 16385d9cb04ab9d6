#!/usr/bin/env python
"""The scene's observers at scale: 2 cameras and 4 reflection probes updated every frame (6 x 4 + 2 = 26 observers).

    (a) fyx_cull_scene_observers, then fyx_pack_scene_observer_instances: one call builds every observer on the device,
        one node pass counts all their lists, one pack packs them;
    (b) what a host does without (a): read the camera and probe nodes' global matrices back (fyx_get_global_matrices),
        then per group of at most 8 observers fyx_set_observers + fyx_cull, fyx_cull_lights and
        fyx_select_reflection_probes, and one fyx_pack_instances per observer.  The observers' matrices are taken once
        from (a)'s table (a host computes them itself from the matrices it read back).
Both routes leave the visible lists and the instances on the device: neither reads them back while it is timed (fyx_pack_instances
is called through the C ABI, without the host copy Context.pack_instances makes).  What each reads back is what its calls need:
(a) the counts its call sizes the lists with, (b) the observers' matrices, each cull's counts and the light lists.

Scene: 10 M nodes from scenegen, with and without LOD ranges (about 1 % of the nodes, three levels) and static batches
(about 0.1 %, nodes with children).  The routes alternate three times in one process, each call timed on the host clock
around work that ends in a synchronise; (a) and (b) must give the same sets.  Prints one JSON line per scene, with the
card's name and power limit read in the same run.

    python tools/observer_bench.py [--nodes 10000000] [--steps 5]
"""
import argparse
import json
import os
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


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:
        return f"unknown ({e})"


def route_a(ctx, read=False):
    ctx.cull_scene_observers(FRAME)
    ctx.pack_scene_observer_instances()
    return ctx.get_scene_observers() if read else None  # the lists stay on the device in both routes; read only to compare


def route_b(ctx, nodes, table, pack=True, read=False):
    ctx.get_global_matrices(nodes)  # the host round trip the device route avoids
    sets, lights, env = [], [], []
    for o0 in range(0, len(table), 8):
        rows = table[o0: o0 + 8]
        ctx.set_observers([(r["translation"], float(r["z_near"]), float(r["z_far"])) for r in rows])
        ctx.cull([fb.frustum_from_view_projection_matrix(r["view_projection"]) or fb.frustum_default() for r in rows],
                 cam_mask=[int(r["render_mask"]) for r in rows])
        ctx.cull_lights()
        if read:  # the lists stay on the device in both routes; read them only to compare
            for f in range(len(rows)):
                sets.append(ctx.get_visible(f))
                lights.append(ctx.get_visible_lights(f))
        env += ctx.select_reflection_probes().tolist()
        if pack:  # through the C ABI: Context.pack_instances would also copy every instance to the host
            for f, r in enumerate(rows):
                view, vp = np.ascontiguousarray(r["view"], f32), np.ascontiguousarray(r["view_projection"], f32)
                ctx._chk(ctx._lib.fyx_pack_instances(ctx._h, f, view.ctypes.data, vp.ctypes.data))
    return sets, lights, env


def same(a, b):
    table, entries, lights = a
    sets, lts, env = b
    return len(table) == len(sets) and all(
        np.array_equal(np.sort(entries[r["first"]: r["first"] + r["count"]]), np.sort(s))
        and np.array_equal(lights[r["lights_first"]: r["lights_first"] + r["lights_count"]], lt)
        and (int(r["kind"]) != fb.OBSERVER_CAMERA or int(r["environment_map"]) == e)
        for r, s, lt, e in zip(table, sets, lts, env))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=10_000_000)
    ap.add_argument("--steps", type=int, default=5)
    args = ap.parse_args()
    gpu = card()
    sc = Scene(args.nodes)
    n = sc.capacity
    rng = np.random.default_rng(11)
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
    lights = np.sort(rng.choice(np.setdiff1d(pool, obs_nodes), 64, replace=False)).astype(np.uint32)
    base = sc.flags.copy()
    base[batches] |= fb.NODE_RENDERABLE
    base[lights] |= fb.NODE_LIGHT
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
        cam[:] = (1, fb.PROJECTION_PERSPECTIVE, 1.2, 0.1, 200.0, (0.0, 0.0))
        ctx.set_cameras(cams, cam)
        pr = np.zeros(4, fb.Context.PROBE_DTYPE)
        pr[:] = (1, fb.PROBE_UPDATE_EACH_FRAME, 0.1, 60.0, (0.0, 0.0, 0.0))
        ctx.set_reflection_probes(probes, pr)
        a = route_a(ctx, read=True)
        table = a[0].copy()
        identical = same(a, route_b(ctx, obs_nodes, table, pack=False, read=True))
        t = {"a": [], "b": []}
        for _ in range(3):  # alternate the routes three times
            for r in ("a", "b"):
                t0 = time.perf_counter()
                for _ in range(args.steps):
                    if r == "a":
                        route_a(ctx)
                    else:
                        route_b(ctx, obs_nodes, table)
                t[r].append((time.perf_counter() - t0) / args.steps * 1e3)
        identical = identical and same(route_a(ctx, read=True), route_b(ctx, obs_nodes, table, pack=False, read=True))
        print(json.dumps({
            "tool": "observer_bench", "scene": name, "gpu": gpu, "nodes": n, "observers": len(table), "entries": int(len(a[1])),
            "light_entries": int(len(a[2])), "lod_objects": int(lod_nodes.size) if pruned else 0,
            "static_batches": int(batches.size) if pruned else 0, "identical_a_b": bool(identical),
            "ms_per_call_a_device": t["a"], "ms_per_call_b_host_route": t["b"],
        }), flush=True)
        ctx.close()


if __name__ == "__main__":
    main()
