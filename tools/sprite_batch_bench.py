"""Times the instance pack of one camera frustum over a scenegen scene with and without sprite / rectangle quad nodes, and an
appearance update of quad records (fyx_set_sprites with unchanged kind, key and layout).

    python tools/sprite_batch_bench.py [--nodes 10000000] [--quads 50000 500000] [--update 100000] [--reps 7]

Prints one JSON line per quad count: the card and its power limit (read in the same run), pack times without and with the
quads (host clock around calls that end in a synchronise, median of --reps), the update's time to a synchronise and that of
the call alone (host checks, staging, enqueue), and per-kernel device times
of one pack with quads from torch.profiler (k_dyn_order and k_dyn_quads apart).  The vertex and triangle bytes written per
pack are given so a rate can be read off the quad kernel's time.  Without a CUDA device it prints "not measured"."""
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
from fyrox_b200 import _lib as L  # noqa: E402
from fyrox_b200.context import Context  # noqa: E402

f32 = np.float32


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True).stdout.strip().splitlines()[0]
    except (OSError, IndexError):
        return ""


def records(rng, n):
    r = np.zeros(n, Context.SPRITE)
    sprite = rng.random(n) < 0.7
    r["kind"] = np.where(sprite, L.SPRITE_3D, L.SPRITE_RECTANGLE)
    r["batch_key"] = np.where(sprite, rng.integers(0, 4, n), rng.integers(4, 8, n))  # four materials per kind
    r["layout_id"] = np.where(sprite, 0, 1)
    r["flip"] = rng.integers(0, 4, n)
    r["uv_rect"] = rng.uniform(0, 1, (n, 4))
    r["size"] = rng.uniform(0.1, 2.0, n)
    r["rotation"] = rng.uniform(-3, 3, n)
    r["color"] = rng.integers(0, 256, (n, 4))
    return r


def kernel_times(fn):
    """Device time per kernel name (ms) of one call of fn, from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        name = e.key
        for k in ("k_dyn_mark", "k_dyn_order", "k_dyn_quads", "k_dyn_geometry", "k_inst_keys", "k_inst_scatter", "k_inst_scan",
                  "k_scatter_words"):
            if k in name:
                t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
                out[k] = out.get(k, 0.0) + t / 1e3
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=10_000_000)
    ap.add_argument("--quads", type=int, nargs="+", default=[50_000, 500_000])
    ap.add_argument("--update", type=int, default=100_000)
    ap.add_argument("--reps", type=int, default=7)
    a = ap.parse_args()
    name = card()
    if not name:
        print(json.dumps({"card": "none", "result": "not measured"}))
        return
    from fyrox_b200.scenegen import Scene

    sc = Scene(a.nodes, n_units=0)
    rng = np.random.default_rng(7)
    ctx = fb.Context()
    ctx.set_topology(sc.parent, sc.flags, sc.render_mask, sc.local_aabb, root=0, global_index=sc.global_index)
    ctx.set_local_matrices(sc.local_m16)
    ctx.update_transforms(fb.UPDATE_ALL)
    ctx.enable_instances()
    # the camera at the origin looking down -z, 60 degrees, z in [0.1, 1000] (column-major)
    fy, zn, zf = 1.0 / np.tan(np.pi / 6), 0.1, 1000.0
    proj = np.zeros((4, 4), f32)
    proj[0, 0], proj[1, 1], proj[2, 2], proj[2, 3], proj[3, 2] = fy / (16 / 9), fy, zf / (zn - zf), zn * zf / (zn - zf), -1.0
    ff = fb.frustum_from_view_projection_matrix(proj.T.reshape(16).copy())
    view = np.eye(4, dtype=f32).reshape(16)
    ctx.cull([ff])
    visible = ctx.get_visible(0)
    renderable = visible[(sc.flags[visible] & fb.NODE_RENDERABLE) != 0]

    def pack():
        ctx._chk(ctx._lib.fyx_pack_instances(ctx._h, 0, view.ctypes.data, view.ctypes.data))  # the pack alone, no read-back

    import torch

    def timed(fn):
        ts = []
        for _ in range(a.reps + 1):
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()  # the whole device: the context's own stream included
            ts.append((time.perf_counter() - t0) * 1e3)
        return float(np.median(ts[1:]))

    without = timed(pack)
    for nq in a.quads:
        nodes = np.sort(rng.choice(renderable, min(nq, renderable.size), replace=False)).astype(np.uint32)
        rec = records(rng, nodes.size)
        ctx.set_sprites(nodes, rec)
        with_q = timed(pack)
        d = ctx.dynamic_batches("frustum", 0)
        vbytes = sum(int(st["vertices"].size) for st in d["streams"].values())
        tbytes = sum(int(st["triangles"].size) * 4 for st in d["streams"].values())
        nu = min(a.update, nodes.size)
        upd_nodes = nodes[:nu].copy()
        upd = rec[:nu].copy()

        def update():
            upd["color"] += np.uint8(1)
            ctx.set_sprites(upd_nodes, upd)

        t_update = timed(update)
        # the call alone: the host checks, the staging copy and the enqueue of one scatter, without waiting for the scatter
        ts = []
        for _ in range(a.reps + 1):
            upd["color"] += np.uint8(1)
            t0 = time.perf_counter()
            ctx.set_sprites(upd_nodes, upd)
            ts.append((time.perf_counter() - t0) * 1e3)
            torch.cuda.synchronize()
        t_call = float(np.median(ts[1:]))
        kt = kernel_times(pack)
        kt_update = kernel_times(update)
        print(json.dumps({"card": name, "nodes": a.nodes, "quads": int(nodes.size), "visible": int(visible.size),
                          "dyn_instances": int(d["instances"].size), "pack_ms_without": without, "pack_ms_with_quads": with_q,
                          "update_records": nu, "update_ms": t_update, "update_call_ms": t_call, "quad_vertex_bytes": vbytes, "quad_triangle_bytes": tbytes,
                          "kernel_ms": kt, "update_kernel_ms": kt_update}), flush=True)
        ctx.clear_sprites()
    ctx.close()
    sc.close()


if __name__ == "__main__":
    main()
