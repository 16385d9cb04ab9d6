"""Every form of k_skin against the oracle (bit for bit) and against the float64 reference of skin_cases (within its
rounding-error bound): the three palette bands (<= 64, 65-128, 129-255 bones), surfaces split into several tiles,
warp tails of every length, blend shapes in every band, zero-vertex surfaces, band changes inside one context, and the
three ways to run a frame (build_palettes + skin, render_prep, two asynchronous render_prep frames in flight).
Every check covers every surface of the context, so a kernel that writes into a neighbour's output is caught."""
import re

import numpy as np
import pytest

import fyrox_b200 as fb
from helpers import bits_equal, cube_frusta
from skin_cases import LAYOUTS, MAX_BLEND_SHAPES, SkinScene, Surf, add_to_context, oracle_skin, reference_of, tile_starts, within

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

BANDS = [1, 63, 64, 65, 100, 127, 128, 129, 200, 254, 255]
COUNTS = [1, 2, 3, 5, 127, 128, 129, 1023, 1024, 1025, 8191, 8192, 8193, 8196, 20003, 33001]
LAYOUT_NAMES = list(LAYOUTS)


def check_all(ctx, sc: SkinScene, sids, what=""):
    """Palettes bit-exact with the oracle's, skinned streams bit-exact with the oracle's and within the float64 bound,
    for every surface of the context."""
    assert len(sids) == len(sc.surfaces)
    for sid, sd in zip(sids, sc.surfaces):
        tag = f"{what} surface {sid} {sd.spec}"
        pal_o = sc.oracle_palette(sd)
        pal_g = ctx.get_palette(sid)
        assert bits_equal(pal_g, pal_o).all(), f"{tag}: palette entries {np.nonzero(~bits_equal(pal_g, pal_o).all(axis=1))[0][:8]} differ"
        if not sd.spec.n_verts:
            continue
        pos_o, nrm_o = oracle_skin(pal_o, sd)
        pos_g, nrm_g = ctx.get_skinned(sid)
        for name, g, o in (("positions", pos_g, pos_o), ("normals", nrm_g, nrm_o)):
            eq = bits_equal(g, o).all(axis=1)
            bad = np.nonzero(~eq)[0]
            assert bad.size == 0, f"{tag}: {name} of {bad.size} vertices differ from the oracle, first {bad[:8]}: {g[bad[:2]]} vs {o[bad[:2]]}"
        ref = reference_of(pal_o, sd)
        for name, g, val, bnd in (("positions", pos_g, ref.pos, ref.pos_bound), ("normals", nrm_g, ref.nrm, ref.nrm_bound)):
            bad = np.nonzero(~within(g, val, bnd).all(axis=1))[0]
            assert bad.size == 0, f"{tag}: {name} of vertices {bad[:8]} outside the float64 bound"


def launched_skin_forms(fn, attempts=3):
    """Palette capacity S (the first template argument: 65, 129 or 257) of every k_skin* kernel that `fn` launches, read
    from a CUDA activity trace of torch.profiler.  The activity records of a short region are occasionally not delivered
    at all; a trace without any k_skin* kernel says nothing about the form, so `fn` (which must be repeatable) is traced
    again, up to `attempts` times.  A trace that does hold skinning kernels is returned as it is."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    forms = []
    for _ in range(attempts):
        with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
            fn()
        names = [e.name for e in prof.events() if e.device_type == DeviceType.CUDA]
        forms = sorted({int(m.group(1)) for m in (re.search(r"k_skin\w*<(\d+),", n) for n in names) if m})
        if forms:
            break
    return forms


def expected_form(max_bones):
    return 65 if max_bones <= 64 else (129 if max_bones <= 128 else 257)


def run_frame(ctx, sc, how, changed=None):
    """One frame by `how`: 'split' (update_transforms + build_palettes + skin) or 'sync' (render_prep)."""
    if how == "split":
        if changed is not None:
            ctx.set_local_matrices(changed[1], changed[0])
        ctx.update_transforms(fb.UPDATE_ALL)
        ctx.build_palettes()
        ctx.skin()
    else:
        kw = {} if changed is None else {"changed_m16": changed[1], "changed_idx": changed[0]}
        ctx.render_prep(update_flags=fb.UPDATE_ALL, frusta=cube_frusta()[1], **kw)


def new_context(sc, specs):
    for s in specs:
        sc.add(s)
    sc.oracle()
    ctx = fb.Context()
    sids = sc.load_into(ctx)
    return ctx, sids


@pytest.mark.parametrize("max_bones", BANDS)
def test_every_band_with_small_palettes_and_blend_shapes_in_one_launch(max_bones):
    """The largest palette picks the kernel form; 1- and 3-bone surfaces run in it too.  A two-tile surface with blend
    shapes, surfaces with and without shapes, every vertex layout, one vertex, warp tails."""
    mb = max_bones
    specs = [
        Surf(mb, 8193, "animated", 7),
        Surf(3, 129, "packed52"),
        Surf(1, 5, "k16", 1),
        Surf(mb, 1, "wide96"),
        Surf(mb, 1025, "animated", 0, extreme=True),
        Surf(min(mb, 40), 127, "k16", MAX_BLEND_SHAPES),
        Surf(mb, 0),
        Surf(2, 3, "wide96", 7),
        Surf(mb, 2050, "packed52", 1, extreme=True),
    ]
    sc = SkinScene(1000 + mb)
    ctx, sids = new_context(sc, specs)
    try:
        assert launched_skin_forms(lambda: run_frame(ctx, sc, "split")) == [expected_form(mb)]
        check_all(ctx, sc, sids, f"max_bones {mb}")
        ctx.set_blend_shape_weights(sids[0], sc.new_weights(sc.surfaces[0]))
        run_frame(ctx, sc, "sync", sc.move_bones(60))
        check_all(ctx, sc, sids, f"max_bones {mb}, frame 2")
    finally:
        ctx.close()


@pytest.mark.parametrize("max_bones,blend", [(64, True), (64, False), (128, True), (255, True)])
def test_tile_splits_and_warp_tails(max_bones, blend):
    """Every vertex count around a warp (128 vertices), a 1024-vertex step and the 8192-vertex tile, up to five tiles;
    the order puts tile starts at many offsets mod 32 and mod 128 groups.  With `blend`, every other surface has blend
    shapes, so shape records are read across tile boundaries (local_quad0 != 0), 128 shapes on a two-tile surface
    (without, every launch takes the form compiled without blend shapes)."""
    rng = np.random.default_rng(max_bones + blend)
    counts = [COUNTS[i] for i in rng.permutation(len(COUNTS))]
    specs = []
    for k, nv in enumerate(counts):
        shapes = 0 if k % 2 or not blend else (MAX_BLEND_SHAPES if nv == 8196 else [1, 7][k % 4 // 2])
        nb = max_bones if k % 3 == 0 else int(rng.integers(1, max_bones + 1))
        specs.append(Surf(nb, nv, LAYOUT_NAMES[k % len(LAYOUT_NAMES)], shapes, extreme=(k % 5 == 4)))
    if blend:
        next(s for s in specs if s.n_verts == 8196).n_shapes = MAX_BLEND_SHAPES
    starts = tile_starts(specs)
    assert len({a % 32 for a, _ in starts}) >= 8 and len({a % 128 for a, _ in starts}) >= 8
    assert sum(1 for _, local in starts if local % 32) >= 3  # tiles that start inside a 128-vertex block of their surface
    sc = SkinScene(2000 + max_bones)
    ctx, sids = new_context(sc, specs)
    try:
        run_frame(ctx, sc, "split")
        check_all(ctx, sc, sids, f"tiles, max_bones {max_bones}")
        run_frame(ctx, sc, "sync", sc.move_bones(80))
        check_all(ctx, sc, sids, f"tiles, max_bones {max_bones}, frame 2")
    finally:
        ctx.close()


def test_zero_vertex_surfaces_with_large_palettes_keep_the_small_band():
    """255- and 200-bone surfaces without vertices (palettes only) next to 64-bone surfaces: the launch stays in the
    <= 64 form, and the palettes of the empty surfaces are still computed."""
    specs = [Surf(255, 0), Surf(64, 5000, "animated"), Surf(200, 0), Surf(64, 8193, "k16"), Surf(255, 0), Surf(17, 129, "packed52"),
             Surf(64, 3, "wide96")]
    sc = SkinScene(3000)
    ctx, sids = new_context(sc, specs)
    try:
        for fr in range(2):
            changed = sc.move_bones(50) if fr else None
            assert launched_skin_forms(lambda: run_frame(ctx, sc, "sync", changed)) == [65]
            check_all(ctx, sc, sids, f"zero-vertex, frame {fr}")
    finally:
        ctx.close()


def test_band_switching_inside_one_context():
    """Frames in the <= 64 form, then a 100-bone surface (65-128 form, the vertex streams grow), then a 200-bone one
    (129-255 form): every earlier surface is re-checked after each addition."""
    sc = SkinScene(4000)
    ctx, sids = new_context(sc, [Surf(64, 5000), Surf(10, 129, "packed52"), Surf(64, 8193, "k16")])
    try:
        for fr in range(2):
            run_frame(ctx, sc, "sync", sc.move_bones(40) if fr else None)
            check_all(ctx, sc, sids, f"<= 64, frame {fr}")
        for spec, form in ((Surf(100, 20003, "animated", 7), 129), (Surf(200, 9000, "wide96", 1, extreme=True), 257), (Surf(64, 5, "k16"), 257)):
            sids.append(add_to_context(ctx, sc, sc.add(spec)))
            changed = sc.move_bones(40)
            assert launched_skin_forms(lambda: run_frame(ctx, sc, "sync", changed)) == [form]
            check_all(ctx, sc, sids, f"after adding {spec}")
            run_frame(ctx, sc, "split", sc.move_bones(40))
            check_all(ctx, sc, sids, f"after adding {spec}, next frame")
    finally:
        ctx.close()


def _async_pair(ctx, sc, ffs, blend_surfaces, sids):
    """Two asynchronous frames in flight (k_palette -> k_skin chained by programmatic dependent launch), bones moved and
    blend-shape weights changed in between; checked once both are collected."""
    pins = []
    for k in range(2):
        idx, m = sc.move_bones(50)
        pm, pi = fb.PinnedBuffer(m.shape, np.float32), fb.PinnedBuffer(idx.shape, np.uint32)
        pm.array[:] = m
        pi.array[:] = idx
        pins.append((pm, pi))
        if blend_surfaces:
            j = blend_surfaces[k % len(blend_surfaces)]
            ctx.set_blend_shape_weights(sids[j], sc.new_weights(sc.surfaces[j]))
        ctx.render_prep(update_flags=fb.UPDATE_ALL, changed_m16=pm.ptr, changed_idx=pi.ptr, n_changed=idx.size, frusta=ffs,
                        readback_visible=True, async_=True)
    ctx.frame_wait()
    ctx.frame_wait()
    ctx.sync()
    for pm, pi in pins:
        pm.free()
        pi.free()


@pytest.mark.parametrize("max_bones", [64, 100, 255])
def test_entry_points_and_frames_in_flight(max_bones):
    """build_palettes + skin, synchronous render_prep, and render_prep(async_=True) with two frames in flight, over the
    same context, with bones moving and blend-shape weights changing between frames."""
    mb = max_bones
    specs = [Surf(mb, 8193, "animated", 7), Surf(mb, 1023, "k16"), Surf(5, 129, "packed52", 1), Surf(mb, 2, "wide96", MAX_BLEND_SHAPES),
             Surf(mb // 2 + 1, 4100, "animated", 0, extreme=True), Surf(mb, 0)]
    sc = SkinScene(5000 + mb)
    ctx, sids = new_context(sc, specs)
    blend = [j for j, s in enumerate(specs) if s.n_shapes]
    ffs = cube_frusta()[1]
    try:
        run_frame(ctx, sc, "split")
        check_all(ctx, sc, sids, "build_palettes + skin")
        ctx.set_blend_shape_weights(sids[0], sc.new_weights(sc.surfaces[0]))
        run_frame(ctx, sc, "sync", sc.move_bones(50))
        check_all(ctx, sc, sids, "render_prep")
        for rep in range(2):
            _async_pair(ctx, sc, ffs, blend, sids)
            check_all(ctx, sc, sids, f"asynchronous pair {rep}")
        run_frame(ctx, sc, "split", sc.move_bones(50))
        check_all(ctx, sc, sids, "build_palettes + skin after asynchronous frames")
    finally:
        ctx.close()


@pytest.mark.parametrize("seed", [1, 2, 3, 4])
def test_seeded_random_mixes(seed):
    """6-20 surfaces drawn from all of the above (palette sizes of every band, vertex counts, layouts, blend shapes,
    overflowing magnitudes), three frames each run by a randomly chosen entry point."""
    rng = np.random.default_rng(seed)
    specs = []
    for _ in range(int(rng.integers(6, 21))):
        nv = int(rng.choice(COUNTS + [0, 0, 4, 64, 500, 4096]))
        if nv > 9000 and rng.random() < 0.6:
            nv = int(rng.integers(1, 3000))
        shapes = int(rng.choice([0, 0, 1, 7, MAX_BLEND_SHAPES])) if nv <= 9000 else int(rng.choice([0, 1, 7]))
        specs.append(Surf(int(rng.choice(BANDS + [2, 3, 17, 40])), nv, str(rng.choice(LAYOUT_NAMES)), shapes, extreme=bool(rng.random() < 0.2)))
    sc = SkinScene(6000 + seed)
    ctx, sids = new_context(sc, specs)
    blend = [j for j, s in enumerate(specs) if s.n_shapes and s.n_verts]
    ffs = cube_frusta()[1]
    try:
        for fr in range(3):
            how = str(rng.choice(["split", "sync", "async"]))
            if how == "async":
                _async_pair(ctx, sc, ffs, blend, sids)
            else:
                if blend:
                    j = blend[fr % len(blend)]
                    ctx.set_blend_shape_weights(sids[j], sc.new_weights(sc.surfaces[j]))
                run_frame(ctx, sc, how, sc.move_bones(30) if fr else None)
            check_all(ctx, sc, sids, f"seed {seed} frame {fr} ({how})")
    finally:
        ctx.close()
