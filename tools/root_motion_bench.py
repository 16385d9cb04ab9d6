"""Times the device animation step with and without signals and root motion, at bench.py's device-animation size (C4:
50 000 animations of 64 UnitQuaternion rotation tracks, 4 linear keys per curve over a 2 s loop).

    python tools/root_motion_bench.py [--units 50000] [--bones 64] [--steps 50] [--reps 5]

Two contexts hold the same scene: each unit is a root node with `bones` children.  In the second, every animation also has
a Position track on its unit root, root-motion settings on that root and 4 signals, and the events are drained after every
frame.  Timed (host clock around calls that end in a synchronise, median of --reps runs alternating the two contexts):
fyx_animate alone, and the asynchronous end-to-end frame (fyx_render_prep with do_animate, two frames in flight, visible
lists read back).  Prints one JSON line with the card and its power limit."""
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

f32 = np.float32
K, T = 4, 2.0


def build(units, bones, features, rng_seed=7):
    rng = np.random.default_rng(rng_seed)
    per = bones + 1
    n = 1 + units * per
    parent = np.zeros(n, np.uint32)
    parent[0] = fb.FYX_NONE
    roots = 1 + np.arange(units, dtype=np.uint32) * per
    for b in range(1, per):
        parent[roots + b] = roots
    flags = np.full(n, fb.NODE_DEFAULT | fb.NODE_RENDERABLE, np.uint32)
    ctx = fb.Context()
    ctx.set_topology(parent, flags, None, np.tile(np.array([-0.5, -0.5, -0.5, 0.5, 0.5, 0.5], f32), (n, 1)))
    trs = np.zeros((n, 10), f32)
    trs[:, 6] = 1.0
    trs[:, 7:10] = 1.0
    trs[roots, 0:2] = rng.uniform(-100, 100, (units, 2))
    trs[roots, 2] = rng.uniform(-200, -5, units)
    ctx.set_local_trs(trs)
    ctx.update_transforms(fb.UPDATE_ALL)
    q = rng.normal(size=(bones, 4, K)).astype(f32)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    nt = bones + (1 if features else 0)
    tracks = np.zeros(nt, fb.Context.TRACK_DTYPE)
    tracks["binding"], tracks["value_kind"], tracks["enabled"] = 2, 5, 1
    tracks["n_curves"], tracks["n_keys"] = 4, K
    tracks["first_key"][:bones] = (np.arange(bones, dtype=np.uint32) * 4 * K)[:, None] + (np.arange(4, dtype=np.uint32) * K)[None, :]
    keys = np.zeros(nt * 4 * K, fb.Context.KEY_DTYPE)
    keys["location"] = np.tile(np.arange(K, dtype=f32) * f32(T / (K - 1)), nt * 4)
    keys["kind"] = 1
    keys["value"][:bones * 4 * K] = q.reshape(-1)
    if features:  # the root's walk: x and z move, y constant
        tracks[bones]["binding"], tracks[bones]["value_kind"], tracks[bones]["n_curves"] = 0, 2, 3
        tracks[bones]["first_key"][:3] = bones * 4 * K + np.arange(3) * K
        keys["value"][bones * 4 * K:bones * 4 * K + 3 * K] = np.concatenate([np.linspace(0, 2, K), np.zeros(K), np.linspace(0, 1, K)]).astype(f32)
    phase = rng.uniform(0.0, T, units).astype(f32)
    for u in range(units):
        tr = tracks.copy()
        tr["target_node"][:bones] = roots[u] + 1 + np.arange(bones, dtype=np.uint32)
        if features:
            tr["target_node"][bones] = roots[u]
        a = ctx.anim_add(tr, keys, speed=1.0, looped=True, time_slice=(0.0, T), time_position=float(phase[u]))
        if features:
            ctx.anim_set_root_motion(a, node=int(roots[u]), ignore_y=True)
            ctx.anim_set_signals(a, [(0.25, True), (0.75, True), (1.25, True), (1.75, True)])
    return ctx


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--units", type=int, default=50_000)
    ap.add_argument("--bones", type=int, default=64)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    ctxs = {"without": build(a.units, a.bones, False), "with": build(a.units, a.bones, True)}
    # a 60-degree perspective camera at the origin looking down -z, z in [0.1, 200] (column-major)
    fy, zn, zf = 1.0 / np.tan(np.pi / 6), 0.1, 200.0
    proj = np.zeros((4, 4), f32)
    proj[0, 0], proj[1, 1], proj[2, 2], proj[2, 3], proj[3, 2] = fy / (16 / 9), fy, zf / (zn - zf), zn * zf / (zn - zf), -1.0
    ff = fb.frustum_from_view_projection_matrix(proj.T.reshape(16).copy())
    dt = 1.0 / 60.0
    events = {"with": 0, "without": 0}

    def animate(name):
        ctx = ctxs[name]
        for _ in range(a.steps):
            ctx.animate(dt)
            if name == "with":
                events[name] += len(ctx.anim_take_events()[0])
        ctx.update_transforms(fb.UPDATE_INCREMENTAL)  # ends in a synchronise

    def frames(name):
        ctx = ctxs[name]
        for i in range(a.steps):
            ctx.render_prep(update_flags=fb.UPDATE_INCREMENTAL, frusta=[ff], do_palettes=False, do_skin=False, readback_visible=True,
                            async_=True, animate_dt=dt)
            if i:
                ctx.frame_wait()
            if name == "with":
                events[name] += len(ctx.anim_take_events()[0])
        ctx.frame_wait()

    res = {}
    for kind, fn in (("animate", animate), ("e2e", frames)):
        fn("without")
        fn("with")  # warm-up of every shape
        ts = {"without": [], "with": []}
        for _ in range(a.reps):
            for name in ("without", "with"):
                t0 = time.perf_counter()
                fn(name)
                ts[name].append((time.perf_counter() - t0) * 1e3 / a.steps)
        res[kind] = {k: float(np.median(v)) for k, v in ts.items()}
    launches = {k: c.kernel_launch_count() for k, c in ctxs.items()}
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"card": card, "units": a.units, "bones": a.bones, "steps": a.steps, "reps": a.reps,
                      "animate_ms_per_frame": res["animate"], "e2e_ms_per_frame": res["e2e"],
                      "extra_animate_ms": res["animate"]["with"] - res["animate"]["without"],
                      "extra_e2e_ms": res["e2e"]["with"] - res["e2e"]["without"],
                      "events_drained": events["with"], "kernel_launches": launches,
                      "timing": "host clock around calls ending in a synchronise; median of alternating runs; the 'with' runs include draining events every frame"}))


if __name__ == "__main__":
    main()
