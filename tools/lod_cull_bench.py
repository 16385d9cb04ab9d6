#!/usr/bin/env python
"""Camera culls of a scene with LOD groups and static batches, at scale: the un-fused cull, where the camera's pruner table
applies the LOD filter and the static-batch pruning.

    update_and_cull: fyx_update_and_cull (every node recomputed, then the pruner table and the cull);
    cull:            fyx_cull over the finished boxes;

each with 1 frustum (a camera) and with 6 (a point light's cube faces), every frustum with its own observer
(fyx_set_observers), so the LOD filter is on.

Scene: 10 M nodes from scenegen, about 1 % LOD objects in three levels and about 0.1 % static batches (nodes with children),
built as tools/shadow_prune_bench.py builds it.  Each case is warmed up to its steady state, then timed with a host clock
around calls that end in a synchronise, over --rounds alternations of the four cases.  Prints one JSON line with the card's
name and power limit read in the same run, and per case the ms per call of each round and a digest of the visible sets.
--lib runs the same cases on another build of the library (same C ABI), so that two builds can be compared by running the
tool once per build, alternating, and comparing the digests.

    python tools/lod_cull_bench.py [--nodes 10000000] [--steps 10] [--rounds 3] [--lib path/to/libfyrox_b200.so]
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import numpy as np  # noqa: E402

import fyrox_b200 as fb  # noqa: E402
from fyrox_b200 import _lib as L  # noqa: E402
from fyrox_b200 import camera  # noqa: E402
from fyrox_b200.scenegen import Scene  # noqa: E402

f32 = np.float32
LEVELS = [(0.0, 0.3), (0.3, 0.8), (0.8, 4.0)]


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:
        return f"unknown ({e})"


def digest(ctx, nf):
    h = hashlib.sha256()
    for f in range(nf):
        h.update(np.sort(ctx.get_visible(f)).tobytes())
        h.update(b"|")
    return h.hexdigest()[:16]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=10_000_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--lib", default=None, help="another build of libfyrox_b200.so")
    args = ap.parse_args()
    if args.lib:
        L.LIB_PATH = os.path.abspath(args.lib)
    gpu = card()
    sc = Scene(args.nodes)
    n = sc.capacity
    rng = np.random.default_rng(7)
    alive = np.flatnonzero(sc.flags & fb.NODE_ALIVE)
    alive = alive[alive > 0]
    n_children = np.bincount(sc.parent[sc.parent != 0xFFFFFFFF].astype(np.int64), minlength=n)
    parents = alive[n_children[alive] > 0]  # scenegen's meshes are leaves: the batches are parents made meshes
    batches = np.sort(rng.choice(parents, min(parents.size, max(1, n // 1000)), replace=False)).astype(np.uint32)
    lod_nodes = np.sort(rng.choice(alive, max(1, n // 100), replace=False)).astype(np.uint32)
    ranges = np.array([LEVELS[k] for k in rng.integers(0, len(LEVELS), lod_nodes.size)], f32)
    flags = sc.flags.copy()
    flags[batches] |= fb.NODE_RENDERABLE | fb.NODE_STATIC_BATCH
    ctx = fb.Context()
    ctx.set_topology(sc.parent, flags, sc.render_mask, sc.local_aabb, root=0)
    ctx.set_local_matrices(sc.local_m16)
    ctx.set_lod_ranges(ranges, lod_nodes)
    ctx.update_transforms(fb.UPDATE_ALL)
    views = {1: ([camera.camera_frustum()], [((0.0, 0.0, 0.0), 0.1, 150.0)]),
             6: (camera.cube_frusta(radius=60.0), [((0.0, 0.0, 0.0), 0.01, 60.0)] * 6)}
    cases = [(call, nf) for call in ("update_and_cull", "cull") for nf in (1, 6)]

    def run(call, nf):
        frusta, obs = views[nf]
        ctx.set_observers(obs)
        if call == "update_and_cull":
            ctx.update_and_cull(frusta, fb.UPDATE_ALL)
        else:
            ctx.cull(frusta)

    ms = {f"{c}_{nf}": [] for c, nf in cases}
    sets, sizes = {}, {}
    for _ in range(args.rounds):
        for call, nf in cases:
            for _ in range(args.warmup):
                run(call, nf)
            t0 = time.perf_counter()
            for _ in range(args.steps):
                run(call, nf)
            ms[f"{call}_{nf}"].append((time.perf_counter() - t0) / args.steps * 1e3)
            d = digest(ctx, nf)
            assert sets.setdefault(f"{call}_{nf}", d) == d, "the visible sets changed between rounds"
            sizes[f"{call}_{nf}"] = [int(ctx.get_visible(f).size) for f in range(nf)]
    print(json.dumps({
        "tool": "lod_cull_bench", "lib": L.LIB_PATH, "gpu": gpu, "nodes": n, "lod_objects": int(lod_nodes.size),
        "static_batches": int(batches.size), "ms_per_call": ms, "visible_digest": sets, "visible_counts": sizes,
    }), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
