"""Times the instance pack of one camera frustum with and without dynamic batching (BatchingMode::Dynamic props).

    python tools/dynamic_batch_bench.py [--nodes 1000000] [--props 50000] [--reps 5]

Prints one JSON line: the card and its power limit, pack times (host clock around calls that end in a synchronise, median
of --reps), the dynamic part's bytes (vertex records read and written, triangles read and written) over its extra time."""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=1_000_000)
    ap.add_argument("--props", type=int, default=50_000)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    rng = np.random.default_rng(1)
    n = a.nodes
    parent = np.zeros(n, np.uint32)
    parent[0] = fb.FYX_NONE
    flags = np.full(n, fb.NODE_DEFAULT | fb.NODE_RENDERABLE, np.uint32)
    local = np.tile(np.eye(4, dtype=f32).reshape(16), (n, 1))
    local[:, 12:14] = rng.uniform(-60, 60, (n, 2))
    local[:, 14] = rng.uniform(-120, -1, n)
    local[0, 12:15] = 0
    ctx = fb.Context()
    ctx.set_topology(parent, flags, np.full(n, 0xFFFFFFFF, np.uint32), np.tile(np.array([-0.5, -0.5, -0.5, 0.5, 0.5, 0.5], f32), (n, 1)))
    ctx.set_local_matrices(local)
    ctx.update_transforms(fb.UPDATE_ALL)
    ctx.enable_instances()
    props = rng.choice(np.arange(1, n), a.props, replace=False)
    layout = (48, 0, 12, 24)
    for k, node in enumerate(props.tolist()):
        nv = int(rng.integers(24, 256))
        v = rng.uniform(-1, 1, (nv, 12)).astype(f32)
        t = rng.integers(0, nv, (nv, 3)).astype(np.uint32)
        ctx.add_dynamic_surface(node, 0, k % 8, 0, layout, v.view(np.uint8).reshape(-1), t)
    # a 60-degree perspective camera at the origin looking down -z, z in [0.1, 200] (column-major)
    fy, zn, zf = 1.0 / np.tan(np.pi / 6), 0.1, 200.0
    proj = np.zeros((4, 4), f32)
    proj[0, 0], proj[1, 1], proj[2, 2], proj[2, 3], proj[3, 2] = fy / (16 / 9), fy, zf / (zn - zf), zn * zf / (zn - zf), -1.0
    ff = fb.frustum_from_view_projection_matrix(proj.T.reshape(16).copy())
    view = np.eye(4, dtype=f32).reshape(16)

    def timed():
        ts = []
        for _ in range(a.reps + 1):
            t0 = time.perf_counter()
            ctx._chk(ctx._lib.fyx_pack_instances(ctx._h, 0, view.ctypes.data, view.ctypes.data))  # the pack alone, no read-back
            ts.append((time.perf_counter() - t0) * 1e3)
        return float(np.median(ts[1:]))

    ctx.cull([ff])
    with_dyn = timed()
    d = ctx.dynamic_batches("frustum", 0)
    st = d["streams"].get(0, {"vertices": np.empty(0), "triangles": np.empty((0, 3))})
    moved = 2 * st["vertices"].size + 2 * 12 * st["triangles"].shape[0]
    ctx.clear_dynamic_surfaces()
    ctx.cull([ff])
    without = timed()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    extra = max(with_dyn - without, 1e-6)
    print(json.dumps({"card": gpu, "nodes": n, "props": a.props, "dyn_instances": int(d["instances"].size), "pack_ms_with_dynamic": with_dyn,
                      "pack_ms_without": without, "dynamic_bytes": int(moved), "dynamic_GBps_over_extra_time": moved / extra / 1e6}))
    ctx.close()


if __name__ == "__main__":
    main()
