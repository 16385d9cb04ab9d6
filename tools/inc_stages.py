#!/usr/bin/env python
"""Stage times (CUDA events of synchronous frames, fyx_get_timings) of the C4 frame in its two update modes, with the changed
bones uploaded every frame: FYX_UPDATE_ALL (every node recomputed) vs FYX_UPDATE_INCREMENTAL (static + skeletons: only the bones
change, clean sub-trees keep matrices and boxes, everything is culled again) — and the pipelined end-to-end time of both.
usage: python tools/inc_stages.py [units]"""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import bench
import fyrox_b200 as fb
from fyrox_b200 import camera
from fyrox_b200.scenegen import Scene


def main():
    units = int(sys.argv[1]) if len(sys.argv) > 1 else 50000
    sc = Scene(units * 200, n_units=units, verts_per_unit=5000, bones_per_unit=64, seed=bench.SEED)
    ctx = fb.Context()
    bench.load_scene(ctx, sc, fb, lambda m: None)
    frusta = camera.cube_frusta()
    n_bones = units * 64
    anim = []
    for fr in range(2):
        pi = fb.PinnedBuffer((n_bones,), np.uint32)
        full_trs = fb.PinnedBuffer((n_bones, 10), np.float32)
        sc.animate_trs_into(fr, pi.ptr, full_trs.ptr)
        if fr == 0:
            ctx.set_local_trs(full_trs.array, pi.array)
        pm = fb.PinnedBuffer((n_bones, 4), np.float32)
        pm.array[:] = full_trs.array[:, 3:7]
        full_trs.free()
        anim.append((pi, pm))
    out = {"units": units}
    for name, flags in (("all_dirty", fb.UPDATE_ALL), ("incremental", fb.UPDATE_INCREMENTAL)):
        acc = {}
        n = 12
        for i in range(n + 3):
            pi, pm = anim[i & 1]
            ctx.render_prep(update_flags=flags, changed_idx=pi.ptr, n_changed=n_bones, changed_rot=pm.ptr, frusta=frusta, readback_visible=False)
            if i >= 3:
                for k, v in ctx.timings().items():
                    if k.endswith("_ms"):
                        acc[k] = acc.get(k, 0.0) + v / n
        # pipelined end to end
        def frames(m):
            for i in range(m):
                pi, pm = anim[i & 1]
                ctx.render_prep(update_flags=flags, changed_idx=pi.ptr, n_changed=n_bones, changed_rot=pm.ptr, frusta=frusta, readback_visible=True, async_=True)
                if i:
                    ctx.frame_wait()
            ctx.frame_wait()
        frames(3)
        ctx.sync()
        t0 = time.perf_counter()
        frames(20)
        ctx.sync()
        acc["pipelined_e2e_ms"] = (time.perf_counter() - t0) * 1e3 / 20
        out[name] = {k: round(v, 4) for k, v in acc.items()}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
