"""The many-map culls (fyx_cull_shadow_casters, _csm, _pruned, fyx_cull_scene_observers, fyx_cull_scene_shadow_casters) share
one sequence: a one-CTA table kernel, the pruner table (one launch per hierarchy level that holds pruners), the count pass,
the scan, and the emit pass when there is a list to write.  Pins the kernel launches of every call in its steady state (the
second call: the first also builds the light table and the pruner column), with and without pruners, and with no map and
no observer at all.  The camera cull (fyx_cull) shares the pruner table's rule: the table (one launch per hierarchy level
that holds pruners), then one launch over all slots."""
import numpy as np
import pytest

import fyrox_b200 as fb
from test_gpu_observers import FRAME, ObserverScene
from test_gpu_scene_shadows import WIDE, shadowy
from test_gpu_shadow_csm import camera

pytestmark = pytest.mark.gpu

f32 = np.float32
OFF = (200.0, 200.0, 0, 0)  # spot and point shadows disabled: without a csm camera no light gets a map


@pytest.fixture(params=[False, True], ids=["no_pruners", "pruners"])
def scene(ctx, request):
    """1500 nodes, 12 shadow-casting lights with large boxes, 3 cameras and 2 probes; with or without LOD objects and static
    batches.  Returns (the scene, the hierarchy levels that hold a pruner)."""
    rng = np.random.default_rng(7700)
    s = ObserverScene(rng, 1500, 3, 2, pruners=request.param)
    shadowy(s)
    sc = s.sc
    sc.load(ctx)  # the camera and probe records are sent by the test
    s.pr.send_ranges(ctx)
    depth = np.zeros(sc.n, np.int64)
    for i in range(1, sc.n):  # a parent comes before its children
        depth[i] = depth[sc.parent[i]] + 1
    pruners = sorted(set(s.pr.ranges) | set(np.flatnonzero((sc.flags & fb.NODE_STATIC_BATCH) != 0).tolist()))
    levels = len({int(depth[x]) for x in pruners})
    assert (levels >= 2) == request.param and (levels == 0) == (not request.param)
    return s, levels


def launches(ctx, fn):
    fn()
    n = ctx.kernel_launch_count()
    fn()
    return ctx.kernel_launch_count() - n


def test_kernel_launches_of_every_map_cull(ctx, scene):
    s, levels = scene
    _, ff, _, fc = camera()
    eye = np.zeros(3, f32)
    ctx.cull([ff])

    def shadow(settings=WIDE, **kw):
        return launches(ctx, lambda: ctx.cull_shadow_casters(0, eye, *settings, **kw))

    def n_entries():
        maps, entries = ctx.get_shadow_maps()
        return len(maps), entries.size

    # the shadow maps of one camera: table, [pruner table,] count, scan, emit
    if not levels:
        assert shadow() == 4
        assert min(n_entries()) > 0
        assert shadow(csm_camera=fc) == 4
        assert min(n_entries()) > 0
    assert shadow(prune=True) == 4 + levels
    assert min(n_entries()) > 0
    assert shadow(csm_camera=fc, prune=True) == 4 + levels
    assert min(n_entries()) > 0
    assert shadow(OFF, prune=True) == 3 + levels  # no map: nothing to emit
    assert n_entries() == (0, 0)

    # no observer: no lists, and no map of theirs
    assert launches(ctx, lambda: ctx.cull_scene_observers(FRAME)) == 5 + levels
    assert len(ctx.get_scene_observers()[0]) == 0
    assert launches(ctx, lambda: ctx.cull_scene_shadow_casters(*WIDE)) == 3 + levels
    assert n_entries() == (0, 0) and len(ctx.get_scene_shadow_maps()) == 0

    # the observers: table, [pruner table,] count, light count, scan, light scan; emit, light emit, light sort; commit
    s.send(ctx)
    assert launches(ctx, lambda: ctx.cull_scene_observers(FRAME)) == 9 + levels
    table, entries, lights = ctx.get_scene_observers()
    assert len(table) > 0 and entries.size > 0 and lights.size > 0
    # their shadow maps: table, [pruner table,] count, scan, emit
    assert launches(ctx, lambda: ctx.cull_scene_shadow_casters(*WIDE)) == 4 + levels
    assert min(n_entries()) > 0 and len(ctx.get_scene_shadow_maps()) > 0



@pytest.mark.parametrize("n_frusta", [1, 6])
def test_kernel_launches_of_a_camera_cull(ctx, scene, n_frusta):
    s, levels = scene
    _, ff, _, _ = camera()
    frusta = [ff] * n_frusta
    ctx.set_observers([((float(k), 0.0, 0.0), 0.1, 150.0) for k in range(n_frusta)])  # the LOD filter is on
    assert launches(ctx, lambda: ctx.cull(frusta)) == 1 + levels
    ctx.set_observers([])  # LOD objects without observers still prune nothing, static batches still do
    assert launches(ctx, lambda: ctx.cull(frusta)) == 1 + levels
