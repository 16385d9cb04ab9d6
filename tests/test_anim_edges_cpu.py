"""The edge cases of tests/anim_edges.py on the CPU: every class is reached and is what it says, the float32 restatement
equals the oracle's curve sampling, time advance, Euler and blend functions bit for bit, both the restatement and the
oracle stay within the float64 bounds, and the float64 check catches self-consistent misreadings of curve.rs that a
comparison with the oracle alone could share."""
import ctypes as C

import numpy as np
import pytest

import anim_edges as ae
import oracle_binding as ob
from helpers import bits_equal

f32 = np.float32


@pytest.fixture(scope="module")
def curves():
    return ae.curve_cases(np.random.default_rng(9001))


@pytest.fixture(scope="module")
def hints():
    return ae.hint_cases(np.random.default_rng(9002))


def test_every_curve_class_is_reached_and_is_what_it_says(curves, hints):
    for c in ae.CURVE_CLASSES:
        assert len(curves[c]) > 0, c
    for c in ae.HINT_CLASSES:
        assert len(hints[c]) > 0, c
    for keys, probes in curves["t_one"]:
        x = probes[0]
        how, li, ri, _ = ae.find_span(keys, x, 0)
        assert how == "search" and x < keys["location"][ri]
        assert ae.span_t(keys[li], keys[ri], x) == f32(1)  # the float32 t rounds to 1 below the key
    assert {int(k["kind"][1]) for k, _ in curves["t_one"]} == {ae.CONST, ae.LIN, ae.CUB}  # the span's left key
    for keys, probes in curves["span_one_ulp"]:
        assert np.nextafter(keys["location"][1], f32(np.inf)) == keys["location"][2]
    for cls, m in (("duplicates_start", 0), ("duplicates_middle", 3), ("duplicates_end", 6)):
        counts = set()
        for keys, probes in curves[cls]:
            d = probes[0]
            counts.add(int((keys["location"] == d).sum()))
            assert (np.diff(keys["location"]) >= 0).all()
            assert keys["location"][m] == d
        assert {2, 3} <= counts, cls
    for keys, probes in curves["large_locations"]:
        assert 1e4 <= keys["location"][0] and keys["location"][-1] <= 1.06e6
    pairs = {(int(k["kind"][0]), int(k["kind"][1])) for k, _ in curves["kind_pairs"]}
    assert len(pairs) == 9
    assert sorted(len(k) for k, _ in curves["key_counts"]) == [0, 1, 2, 3, 31, 32, 33, 1000, 70000]
    over = [ae.curve_value_at(k, x)[0] for k, ps in curves["overflow"] for x in ps]
    assert not np.isfinite(over).all()
    for keys, probes in curves["on_key"]:
        assert np.isin(probes, keys["location"]).all()
    for keys, ts in hints["key_after_left_span"] + hints["key_after_right_span"]:
        j = int(np.nonzero(keys["location"] == ts[1])[0][0])
        assert ae.lerp_one_differs(keys["value"][j - 1], keys["value"][j])
        # the two visits of the key give the two expressions: t = 1 of the left span, t = 0 of the right one
        h = 0
        seen = []
        for t in ts:
            v, h2 = ae.curve_value_at(keys, t, h)
            seen.append((ae.find_span(keys, t, h)[0], v))
            h = h2
        assert {seen[1][0], seen[3][0]} == {"search", "hint"} and seen[1][1] != seen[3][1]


def test_every_time_and_blend_class_is_reached_and_is_what_it_says():
    cases = ae.time_cases()
    classes = {c[0] for c in cases}
    assert classes == set(ae.TIME_CLASSES)
    for case in cases:
        cls, name, (lo, hi), looped, t0, s = case
        n = ae.first_n(case)
        ln = f32(hi - lo)
        if cls == "on_end":
            assert n == hi
        elif cls == "end_ulp_below":
            assert n == np.nextafter(hi, f32(-np.inf))
        elif cls == "end_ulp_above":
            assert n == np.nextafter(hi, f32(np.inf))
        elif cls == "on_start_plus_k_len":
            assert any(n == f32(lo + f32(f32(k) * ln)) for k in ae.K_LENS)
        elif cls.startswith("q_2_") and ln > 0:
            q = abs(float(n - lo) / float(ln))
            e = int(cls[4:])
            assert 2 ** e - 3 <= q <= 2 ** e + 3, (case, q)
        elif cls == "negative":
            assert n < 0
    names = {c[1] for c in cases}
    assert names == set(ae.TIME_SLICES)
    bl = ae.blend_cases(np.random.default_rng(5))
    for c in ae.BLEND_CLASSES:
        assert bl[c], c
    for is_quat, a, b, w in bl["dot_plus_zero"]:
        d = ae._dot4(a, b)
        assert d == 0 and not np.signbit(d)
    for is_quat, a, b, w in bl["dot_minus_zero"]:
        d = ae._dot4(a, b)
        assert d == 0 and np.signbit(d)
    assert {float(w) for _, _, _, w in bl["weights"]} == {float(f32(w)) for w in ae.BLEND_WEIGHTS}
    eu = ae.euler_cases(np.random.default_rng(6))
    assert np.abs(np.concatenate(eu["around_1e6"])).min() > 105615  # above glibc / CUDA's fast range-reduction bound


def test_float32_restatement_equals_the_oracle(curves, hints):
    n = 0
    for cls, cases in curves.items():
        for keys, probes in cases:
            for x in probes:
                for hint in sorted({0, 1, len(keys) // 2, max(len(keys) - 1, 0), len(keys), len(keys) + 3}):
                    want, wh = ob.curve_value_at(keys, float(x), hint)
                    got, gh = ae.curve_value_at(keys, x, hint)
                    assert ae.same_bits(got, want) and gh == wh, (cls, x, hint, got, want)
                    n += 1
            if len(keys) >= 2:
                for i in range(len(keys) - 1):
                    if i > 40:
                        break
                    for t in (0.0, 0.25, 0.5, 1.0, float(np.nextafter(f32(1), f32(0)))):
                        assert ae.same_bits(ae.key_interpolate(keys[i], keys[i + 1], t), ae.oracle_key_interpolate(keys[i], keys[i + 1], t)), (cls, i, t)
    for cls, cases in hints.items():
        for keys, ts in cases:
            h0, h1 = 0, C.c_uint32(0)
            for t in ts:
                got, h0 = ae.curve_value_at(keys, t, h0)
                want = ob.lib().orc_curve_value_at(keys.ctypes.data_as(C.c_void_p), len(keys), float(t), C.byref(h1))
                assert ae.same_bits(got, want) and h0 == h1.value, (cls, t)
    assert n > 3000
    for case in ae.time_cases():
        _, _, (lo, hi), _, t0, s = case
        for x in (ae.first_n(case), t0, f32(t0 - s)):
            assert ae.same_bits(ae.wrapf(x, lo, hi), ob.lib().orc_wrapf(float(x), float(lo), float(hi))), (case, x)
    for cls, es in ae.euler_cases(np.random.default_rng(6)).items():
        for e in es:
            assert bits_equal(ae.quat_from_euler_xyz(e), ae.oracle_quat_from_euler(e)).all(), (cls, e)
    for cls, cs in ae.blend_cases(np.random.default_rng(5)).items():
        for is_quat, a, b, w in cs:
            assert bits_equal(ae.track_value_blend(is_quat, a, b, w), ae.oracle_blend(is_quat, a, b, w)).all(), (cls, a, b, w)


def curve_errors(curves, value_at, fail_fast=False):
    """(largest error / bound, cases checked, cases skipped) of `value_at` against the float64 curve over every probe
    and every hint; with fail_fast, returns at the first violation."""
    worst, checked, skipped = 0.0, 0, 0
    for cls, cases in curves.items():
        for keys, probes in cases:
            for x in probes:
                for hint in sorted({0, len(keys) // 2, len(keys)}):
                    want, bound = ae.curve_value_at64(keys, x, hint)
                    if bound is None:
                        skipped += 1
                        continue
                    got = float(value_at(keys, x, hint)[0])
                    err = abs(got - want) if np.isfinite(got) else np.inf
                    checked += 1
                    if err > bound:
                        if fail_fast:
                            return np.inf, checked, skipped
                        raise AssertionError((cls, x, hint, got, want, bound))
                    if bound > 0:
                        worst = max(worst, err / bound)
    return worst, checked, skipped


def test_float32_paths_are_within_the_float64_bounds(curves, hints):
    worst, checked, skipped = curve_errors(curves, ae.curve_value_at)
    assert checked > 2000 and skipped < checked / 4
    print(f"curves: largest error / bound {worst:.3f} over {checked} cases, {skipped} skipped")
    for cls, cases in hints.items():
        for keys, ts in cases:
            h = 0
            for t in ts:
                want, bound = ae.curve_value_at64(keys, t, h)
                got, h = ae.curve_value_at(keys, t, h)
                assert bound is None or abs(float(got) - want) <= bound, (cls, t)
    worst = 0.0
    n_skip = 0
    for case in ae.time_cases():
        cls, _, (lo, hi), looped, t0, s = case
        n = ae.first_n(case)
        bound = ae.wrap_bound(n, lo, hi)
        if bound is None:
            n_skip += 1
            continue
        d = ae.phase_distance(ae.wrapf(n, lo, hi), ae.wrapf64(n, lo, hi), lo, hi)
        d_or = ae.phase_distance(ob.lib().orc_wrapf(float(n), float(lo), float(hi)), ae.wrapf64(n, lo, hi), lo, hi)
        assert d <= bound and d_or <= bound, (case, n, d, bound)
        if bound:
            worst = max(worst, d / bound)
    print(f"wrapf: largest phase error / bound {worst:.3f}, {n_skip} skipped (|n / len| >= 2^24 or len = 0)")
    worst_q = worst_m = 0.0
    for cls, es in ae.euler_cases(np.random.default_rng(6)).items():
        for e in es:
            q64 = ae.quat_from_euler64(e)
            q = ae.oracle_quat_from_euler(e).astype(np.float64)
            worst_q = max(worst_q, np.abs(q - q64).max() / ae.EULER_QUAT_BOUND)
            tr = ob.Transform()
            ob.lib().orc_transform_identity(C.byref(tr))
            tr.local_rotation[:] = ae.oracle_quat_from_euler(e).tolist()
            m = np.empty(16, np.float32)
            ob.lib().orc_transform_calculate_local(C.byref(tr), ob.fp(m))
            R = m[[0, 1, 2, 4, 5, 6, 8, 9, 10]].astype(np.float64)
            worst_m = max(worst_m, np.abs(R - ae.rotation_matrix64(q64)).max() / ae.EULER_MAT_BOUND)
    assert worst_q <= 1 and worst_m <= 1, (worst_q, worst_m)
    print(f"euler: largest quaternion error / bound {worst_q:.3f}, matrix {worst_m:.3f}")
    worst = 0.0
    for cls, cs in ae.blend_cases(np.random.default_rng(5)).items():
        for is_quat, a, b, w in cs:
            want, bound = ae.track_value_blend64(is_quat, a, b, w)
            if want is None:
                continue
            got = ae.track_value_blend(is_quat, a, b, w).astype(np.float64)
            err = np.abs(got - want)
            assert (err <= bound).all(), (cls, a, b, w, got, want)
            worst = max(worst, float((err / np.maximum(bound, 1e-300)).max()))
    print(f"blend: largest error / bound {worst:.3f}")


# ---- the float64 check catches misreadings the oracle comparison could share ----------------------------------------

def _interp_swapped_tangents(l, r, t):
    if int(l["kind"]) != ae.CUB:
        return ae.key_interpolate(l, r, t)
    m1 = r["left_tangent"] if int(r["kind"]) == ae.CUB else 0.0
    return ae.cubicf(l["value"], r["value"], t, m1, l["right_tangent"])


def _interp_right_family(l, r, t):
    return ae.key_interpolate({**{n: l[n] for n in ae.KD.names}, "kind": r["kind"]}, r, t)


def _interp_no_scale(l, r, t):
    if int(l["kind"]) != ae.CUB:
        return ae.key_interpolate(l, r, t)
    p0, p1, t = f32(l["value"]), f32(r["value"]), f32(t)
    m0, m1 = f32(l["right_tangent"]), f32(r["left_tangent"] if int(r["kind"]) == ae.CUB else 0.0)
    h = lambda a, b, c, d: f32(f32(a * t ** 3) + f32(b * t * t)) + f32(c * t) + f32(d)
    return f32(h(2, -3, 0, 1) * p0 + h(1, -2, 1, 0) * m0 + h(-2, 3, 0, 0) * p1 + h(1, -1, 0, 0) * m1)


def _value_at(interp, span_shift=0):
    def value_at(keys, x, hint):
        if len(keys) == 0:
            return f32(0), hint
        how, li, ri, h = ae.find_span(keys, x, hint)
        if how in ("first", "last"):
            return f32(keys[li]["value"]), h
        if span_shift and ri + 1 < len(keys):
            li, ri = li + 1, ri + 1
        return interp(keys[li], keys[ri], ae.span_t(keys[li], keys[ri], x)), h
    return value_at


@pytest.mark.parametrize("mutant", ["swap_m0_m1", "family_from_right_key", "drop_scale", "next_span"])
def test_float64_check_catches_a_self_consistent_misreading(curves, mutant):
    value_at = {"swap_m0_m1": _value_at(_interp_swapped_tangents), "family_from_right_key": _value_at(_interp_right_family),
                "drop_scale": _value_at(_interp_no_scale), "next_span": _value_at(ae.key_interpolate, span_shift=1)}[mutant]
    worst, _, _ = curve_errors(curves, value_at, fail_fast=True)
    assert worst == np.inf, mutant


# ---- Transform::dirty over one frame -----------------------------------------------------------------------------

def test_one_frame_keeps_transforms_dirty_across_player_and_machine():
    """Graph::update runs the player and the machine in one node loop with no matrix() between them: the machine's -0
    is stored because the player left the transform dirty.  The global matrix shows the sign."""
    parent, trs, (td, kd), (tg, kg) = ae.zero_scale_pair()
    results = []
    for shared in (True, False):
        local = np.empty((3, 16), np.float32)
        tr = ae.oracle_transforms(trs)
        for i in range(3):
            ob.lib().orc_transform_calculate_local(C.byref(tr[i]), ob.fp(local[i]))
        og = ob.Graph.build(parent, None, None, local, None)
        og.update_hierarchical_data()
        direct, src = ob.Animation(td, kd, time_slice=(0.0, 1.0)), ob.Animation(tg, kg, time_slice=(0.0, 1.0))
        ob.update_animations([direct], 0.1, og, tr)
        if not shared:
            og.update_hierarchical_data()  # what a matrix() between the passes would do
        ob.blend_group_update([src], [1.0], 0.1, og, tr)
        og.update()
        results.append((tr[2].local_scale[0], og.global_transform(2)))
    (s_shared, g_shared), (s_apart, g_apart) = results
    assert np.signbit(f32(s_shared)) and not np.signbit(f32(s_apart))
    assert not bits_equal(g_shared, g_apart).all()
