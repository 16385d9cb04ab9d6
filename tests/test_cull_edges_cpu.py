"""The edge boxes of tests/cull_edges.py on the CPU: every class is reached for every frustum shape, the literal restatement equals
the oracle's Frustum::is_intersects_aabb on every box, and so does the numpy form of the kernels' predicate (max corner by the
sign of the normal component, the pm reject, the distinct-coordinate masks including the n_ax > 4 half, the literal path for
non-tame boxes)."""
import numpy as np
import pytest

import cull_edges as ce

f32 = np.float32


@pytest.fixture(scope="module")
def frusta_and_boxes():
    rng = np.random.default_rng(4242)
    frusta = ce.edge_frusta(rng)
    return [(ef, ce.edge_boxes(ef, rng)) for ef in frusta]


def test_every_class_is_reached_for_every_frustum_shape(frusta_and_boxes):
    names = [ef.name for ef, _ in frusta_and_boxes]
    assert {"perspective0", "cube(1, 0, 0)", "ortho_cascade", "far_thin", "corners_off_planes", "nan_corner"} <= set(names)
    for ef, cls in frusta_and_boxes:
        pm_free = np.isnan(ce.dev_frustum_pm(ef.planes, ef.corners)).all()  # a NaN corner makes every pm NaN: no pm edge exists
        for c in ce.CLASSES:
            if pm_free and c.startswith("pm_"):
                continue
            assert len(cls[c]) > 0, (ef.name, c)
        # each class is what it says, box by box, and none has thinned out
        lab = ce.classify(ef.planes, ef.corners, np.concatenate(list(cls.values())))
        for c in ce.CLASSES:
            assert ce.classify(ef.planes, ef.corners, cls[c])[c].all(), (ef.name, c)
        for c in ("corner_on", "corner_in", "corner_out"):
            assert len(cls[c]) >= (8 if ef.name != "nan_corner" else 7) * 3 - (8 if c == "corner_out" else 0), (ef.name, c, len(cls[c]))
        assert lab["fallback_true"].sum() > 0, ef.name
        # the rotated perspectives have 8 distinct coordinates per axis: corners 4..7 sit in the second half of the lists
        if ef.name.startswith("perspective"):
            assert lab["fallback_late_coord"].sum() > 0, ef.name


def test_boundary_classes_sit_exactly_on_their_boundary(frusta_and_boxes):
    for ef, cls in frusta_and_boxes:
        s = ce.max_corner_s(ef.planes, np.concatenate([cls["plane_zero"], cls["point_plane"]]))
        assert ((s == 0).any(1)).all(), ef.name
        pm = ce.dev_frustum_pm(ef.planes, ef.corners)
        if len(cls["pm_equal"]):
            assert (ce.max_corner_s(ef.planes, cls["pm_equal"]) == pm[None]).any(1).all(), ef.name
            assert (ce.max_corner_s(ef.planes, cls["pm_below"]) < pm[None]).any(1).all(), ef.name
        # the ulp variants of a box on a corner: the corner strictly inside one way, outside the other
        inside = lambda b: np.stack([((c >= b[:, :3]) & (c <= b[:, 3:])).all(1) for c in ef.corners], 1).any(1)
        assert inside(cls["corner_on"]).all() and inside(cls["corner_in"]).all(), ef.name
        assert inside(cls["point_corner"]).all(), ef.name
        assert not ce.is_tame(cls["non_tame"]).any()


def test_literal_restatement_equals_the_oracle(frusta_and_boxes):
    total = 0
    for ef, cls in frusta_and_boxes:
        for c, boxes in cls.items():
            want = ce.oracle_aabb_intersects(ef.fo, boxes)
            got = ce.literal_intersects(ef.planes, ef.corners, boxes)
            assert np.array_equal(got, want), (ef.name, c, boxes[got != want][:3])
            total += len(boxes)
            # both answers occur near every boundary, so neither side of an edge goes untested
        both = ce.literal_intersects(ef.planes, ef.corners, np.concatenate([cls["corner_on"], cls["corner_out"], cls["plane_zero"],
                                                                            cls["plane_above"]]))
        assert both.any() and not both.all(), ef.name
    assert total > 2000


def test_kernel_form_gives_the_literal_booleans(frusta_and_boxes):
    for ef, cls in frusta_and_boxes:
        boxes = np.concatenate(list(cls.values()))
        want = ce.literal_intersects(ef.planes, ef.corners, boxes)
        got = ce.kernel_intersects(ef.planes, ef.corners, boxes)
        assert np.array_equal(got, want), (ef.name, boxes[got != want][:3])
        # every box against every other shape as well (a box made for one frustum is an arbitrary box to the next)
        for other, _ in frusta_and_boxes:
            assert np.array_equal(ce.kernel_intersects(other.planes, other.corners, boxes),
                                  ce.literal_intersects(other.planes, other.corners, boxes)), (ef.name, other.name)


def test_interleave_puts_non_tame_boxes_in_every_warp():
    rng = np.random.default_rng(3)
    frusta = ce.edge_frusta(rng)[:2]
    boxes = ce.all_boxes(frusta, rng)
    tame = ce.is_tame(boxes)
    n_warps = len(boxes) // 32
    per_warp = [(~tame[w * 32:(w + 1) * 32]).sum() for w in range(n_warps)]
    assert n_warps > 10 and all(2 <= k <= 8 for k in per_warp), per_warp
