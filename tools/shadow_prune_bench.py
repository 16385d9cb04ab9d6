#!/usr/bin/env python
"""Shadow-caster culls of a scene with LOD groups and static batches, at scale.

    (a) fyx_cull_shadow_casters_pruned on the scene: every map with its own LOD filter and static-batch pruning;
    (b) fyx_cull_shadow_casters_csm on the same scene without its ranges and batch flags (a context of its own): what the
        pruning costs on the device;
    (c) what a host does without (a): the map table (taken once from fyx_get_shadow_maps; a host computes it itself), then
        fyx_cull with at most 8 maps per call, each map's observer sent through fyx_set_observers, every list read back.

Scene: 10 M nodes from scenegen, about 1 % LOD objects in three levels and about 0.1 % static batches (nodes with children),
light nodes among them in front of the camera.  Two loads: 8 spot + 8 point lights (56 maps) and 32 point lights (192 maps).
The routes run in one process and alternate three times; (a) and (c) must give the same sets.  Each timed call starts
from the camera cull.  Prints one JSON line per load, with the card's name and power limit read in the same run.

    python tools/shadow_prune_bench.py [--nodes 10000000] [--steps 5]
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
from fyrox_b200 import camera  # noqa: E402
from fyrox_b200.scenegen import Scene  # noqa: E402

f32 = np.float32
SETTINGS = (60.0, 60.0, 1, 1)  # spot / point shadows_distance, enabled
LEVELS = [(0.0, 0.3), (0.3, 0.8), (0.8, 4.0)]


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:
        return f"unknown ({e})"


def load(ctx, sc, flags):
    ctx.set_topology(sc.parent, flags, sc.render_mask, sc.local_aabb, root=0)
    ctx.set_local_matrices(sc.local_m16)
    ctx.update_transforms(fb.UPDATE_ALL)


def route_a(ctx, cam_ff, cam_t, prune, copy=True):
    ctx.set_observers([])
    ctx.cull([cam_ff])
    ctx.cull_shadow_casters(0, cam_t, *SETTINGS, prune=prune)
    return ctx.get_shadow_maps(copy=copy)


def map_observers(ctx, maps, sources):
    """The map's observer of the reference's from_graph: the light's position, z_near 0.01, z_far light_radius (unit scale)."""
    g = ctx.get_global_matrices(np.array([int(m["light"]) for m in maps], np.uint32)) if len(maps) else np.zeros((0, 16), f32)
    return [(tuple(g[k, 12:15].tolist()), 0.01, float(f32(sources[int(m["light"])][2]))) for k, m in enumerate(maps)]


def route_c(ctx, cam_ff, vps, obs, copy=True):
    ctx.set_observers([])
    ctx.cull([cam_ff])
    lists = []
    for b in range(0, len(vps), 8):
        frusta = [fb.frustum_from_view_projection_matrix(vp) or fb.frustum_default() for vp in vps[b: b + 8]]
        ctx.set_observers(obs[b: b + 8])
        ctx.cull(frusta, pass_flags=[fb.PASS_SHADOW] * len(frusta))
        lists += [ctx.get_visible(k, copy=copy) for k in range(len(frusta))]
    return lists


def same(a, lists):
    maps, entries = a
    return len(maps) == len(lists) and all(
        np.array_equal(np.sort(entries[m["first"]: m["first"] + m["count"]]), np.sort(lst)) for m, lst in zip(maps, lists))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=10_000_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--radius", type=float, default=8.0)
    args = ap.parse_args()
    gpu = card()
    sc = Scene(args.nodes)
    n = sc.capacity
    rng = np.random.default_rng(7)
    alive = np.flatnonzero(sc.flags & fb.NODE_ALIVE)
    alive = alive[alive > 0]
    n_children = np.bincount(sc.parent[sc.parent != 0xFFFFFFFF].astype(np.int64), minlength=n)
    parents = alive[n_children[alive] > 0]  # scenegen's meshes are leaves: the batches are parents made meshes (in both scenes)
    batches = np.sort(rng.choice(parents, min(parents.size, max(1, n // 1000)), replace=False)).astype(np.uint32)
    lod_nodes = np.sort(rng.choice(alive, max(1, n // 100), replace=False)).astype(np.uint32)
    ranges = np.array([LEVELS[k] for k in rng.integers(0, len(LEVELS), lod_nodes.size)], f32)
    plain = sc.flags.copy()
    plain[batches] |= fb.NODE_RENDERABLE
    pruned = plain.copy()
    pruned[batches] |= fb.NODE_STATIC_BATCH
    ctx, ctx_b = fb.Context(), fb.Context()
    load(ctx, sc, pruned)
    ctx.set_lod_ranges(ranges, lod_nodes)
    load(ctx_b, sc, plain)
    cam_t = np.zeros(3, f32)
    cand = rng.choice(np.flatnonzero(plain & fb.NODE_RENDERABLE), 20000, replace=False).astype(np.uint32)
    pos = ctx.get_global_matrices(cand)[:, 12:15]
    gvis = fb.NODE_GLOBAL_VISIBILITY | fb.NODE_GLOBAL_ENABLED
    ok = ((ctx.get_global_flags(cand) & gvis) == gvis) & (pos[:, 2] < -8) & (pos[:, 2] > -50) & (np.abs(pos[:, 0]) < 0.3 * -pos[:, 2]) & (np.abs(pos[:, 1]) < 0.3 * -pos[:, 2])
    pool = np.setdiff1d(np.sort(cand[ok]), np.concatenate([batches, lod_nodes]))
    for name, n_spot, n_point in (("8 spot + 8 point", 8, 8), ("32 point", 0, 32)):
        lights = np.sort(rng.choice(pool, n_spot + n_point, replace=False)).astype(np.uint32)
        kinds = np.array([fb.LIGHT_SPOT] * n_spot + [fb.LIGHT_POINT] * n_point)[rng.permutation(n_spot + n_point)]
        sources = {int(x): (int(k), float(f32(1.0)), float(f32(args.radius))) for x, k in zip(lights, kinds)}
        rec = np.zeros(len(lights), fb.Context.LIGHT_SOURCE_DTYPE)
        for k, x in enumerate(lights.tolist()):
            rec[k] = sources[x]
        for c, fl in ((ctx, pruned), (ctx_b, plain)):
            f2 = fl.copy()
            f2[lights] |= fb.NODE_LIGHT | fb.NODE_CAST_SHADOWS
            c.set_flags(f2[lights], lights)
            c.update_transforms(fb.UPDATE_ALL)
            c.set_light_sources(rec, lights)
        cam_ff = camera.camera_frustum()
        a = route_a(ctx, cam_ff, cam_t, True)
        maps = a[0]
        vps = [m["view_projection"].copy() for m in maps]
        obs = map_observers(ctx, maps, sources)
        identical = same(a, route_c(ctx, cam_ff, vps, obs))
        b = route_a(ctx_b, cam_ff, cam_t, False)
        key = lambda t: [(int(m["light"]), int(m["face"]), int(m["cascade"]), m["view_projection"].tobytes()) for m in t]  # noqa: E731
        same_table = key(b[0]) == key(maps)  # the lists' places differ: pruning shortens them
        t = {"a": [], "b": [], "c": []}
        for _ in range(3):  # alternate the routes three times
            for r in ("a", "b", "c"):
                t0 = time.perf_counter()
                for _ in range(args.steps):
                    if r == "a":
                        route_a(ctx, cam_ff, cam_t, True, copy=False)
                    elif r == "b":
                        route_a(ctx_b, cam_ff, cam_t, False, copy=False)
                    else:
                        route_c(ctx, cam_ff, vps, obs, copy=False)
                t[r].append((time.perf_counter() - t0) / args.steps * 1e3)
        a = route_a(ctx, cam_ff, cam_t, True)
        identical = identical and same(a, route_c(ctx, cam_ff, vps, obs))
        b_entries = int(len(route_a(ctx_b, cam_ff, cam_t, False)[1]))
        print(json.dumps({
            "tool": "shadow_prune_bench", "load": name, "gpu": gpu, "nodes": n, "maps": len(maps), "lod_objects": int(lod_nodes.size),
            "static_batches": int(batches.size), "entries_a": int(len(a[1])), "entries_b": b_entries,
            "identical_a_c": bool(identical), "same_table_a_b": bool(same_table),
            "ms_per_call_a_pruned": t["a"], "ms_per_call_b_unpruned": t["b"], "ms_per_call_c_host_route": t["c"],
        }), flush=True)
        for c, fl in ((ctx, pruned), (ctx_b, plain)):  # the next load starts without these lights
            c.set_light_sources(np.zeros(len(lights), fb.Context.LIGHT_SOURCE_DTYPE), lights)
            c.set_flags(fl[lights], lights)
    ctx.close()
    ctx_b.close()


if __name__ == "__main__":
    main()
