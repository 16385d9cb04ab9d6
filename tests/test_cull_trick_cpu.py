"""The cull kernels do not run the reference's 8 corners x 6 planes loop (fyrox-math/src/frustum.rs:205-219): they test, per
plane, the ONE corner built from the per-axis bound whose product with the normal component is the larger one, and claim
identical booleans because IEEE rounding is monotone (fyx_math.cuh, frustum_intersects_aabb).  This file checks that claim
on the CPU, in numpy float32 (one rounding per operation, like the kernels' __fmul_rn / __fadd_rn), over millions of random
and adversarial planes / boxes — including zeros of both signs, denormals, huge and tiny magnitudes, degenerate boxes — and
the same for the corner-in-box fallback evaluated through per-axis masks of DISTINCT corner coordinates."""
import numpy as np

f32 = np.float32


def s_of(n, d, px, py, pz):
    """Plane::dot + d in the reference's order: ((nx*px + ny*py) + nz*pz) + d, one rounding per op."""
    return ((n[:, 0] * px + n[:, 1] * py) + n[:, 2] * pz) + d


def literal_all_behind(n, d, lo, hi):
    """all 8 corners have s <= 0 (frustum.rs:208-214 for one plane)"""
    allb = np.ones(len(n), bool)
    for c in range(8):
        px = np.where(c & 1, hi[:, 0], lo[:, 0])
        py = np.where(c & 2, hi[:, 1], lo[:, 1])
        pz = np.where(c & 4, hi[:, 2], lo[:, 2])
        allb &= s_of(n, d, px, py, pz) <= 0
    return allb


def trick_all_behind(n, d, lo, hi):
    """the kernels' form: operand picked by the sign of the normal component (n < 0 -> min, else max), one corner"""
    vx = np.where(n[:, 0] < 0, lo[:, 0], hi[:, 0])
    vy = np.where(n[:, 1] < 0, lo[:, 1], hi[:, 1])
    vz = np.where(n[:, 2] < 0, lo[:, 2], hi[:, 2])
    return s_of(n, d, vx, vy, vz) <= 0


def special_values(rng, m):
    pool = np.array([0.0, -0.0, 1.0, -1.0, 0.5, -0.5, 1e-45, -1e-45, 1e-38, -1e-38, 1e-20, 3.0, -3.0, 1e10, -1e10, 1e17, -1e17, 0.1, -0.1,
                     1.0000001, 0.99999994, 16777216.0, -16777217.0, 1e-7, -1e-7], f32)
    return pool[rng.integers(0, len(pool), m)]


def make_cases(rng, m, mode):
    if mode == "random":
        n = rng.normal(size=(m, 3)).astype(f32)
        d = (rng.normal(size=m) * 10).astype(f32)
        a = (rng.normal(size=(m, 3)) * 20).astype(f32)
        b = (rng.normal(size=(m, 3)) * 20).astype(f32)
    elif mode == "scaled":  # wildly different magnitudes per component: cancellation and absorption everywhere
        e = lambda *s, top=12: (10.0 ** rng.uniform(-12, top, s)).astype(f32)
        # plane normals are unit vectors in the engine; here up to 1e6 so that no product overflows (|n|*|bound| <= 1e24):
        # the claim is about rounding, not about inf - inf
        n = (rng.normal(size=(m, 3)).astype(f32)) * e(m, 3, top=5)
        d = rng.normal(size=m).astype(f32) * e(m)
        a = rng.normal(size=(m, 3)).astype(f32) * e(m, 3)
        b = rng.normal(size=(m, 3)).astype(f32) * e(m, 3)
    else:  # "special": zeros of both signs, denormals, ties
        n = special_values(rng, m * 3).reshape(m, 3)
        d = special_values(rng, m)
        a = special_values(rng, m * 3).reshape(m, 3)
        b = special_values(rng, m * 3).reshape(m, 3)
    lo, hi = np.minimum(a, b), np.maximum(a, b)
    # the kernels take this path only for "tame" boxes (finite, |bound| <= 1e18, min <= max); -0/+0 pairs count as ordered
    keep = (np.abs(lo) <= 1e18).all(1) & (np.abs(hi) <= 1e18).all(1)
    return n[keep], d[keep], lo[keep], hi[keep]


def test_max_corner_equals_the_eight_corner_loop():
    rng = np.random.default_rng(2024)
    total = 0
    with np.errstate(over="ignore", under="ignore", invalid="ignore"):
        for mode, m in (("random", 2_000_000), ("scaled", 2_000_000), ("special", 2_000_000)):
            n, d, lo, hi = make_cases(rng, m, mode)
            a, b = literal_all_behind(n, d, lo, hi), trick_all_behind(n, d, lo, hi)
            assert np.isfinite(s_of(n, d, hi[:, 0], hi[:, 1], hi[:, 2])).all()
            assert np.array_equal(a, b), (mode, int((a != b).sum()), n[a != b][:3], d[a != b][:3], lo[a != b][:3], hi[a != b][:3])
            total += len(n)
    assert total > 5_000_000


def test_corner_in_box_through_distinct_coordinate_masks():
    """Fallback of Frustum::is_intersects_aabb (frustum.rs:238-243): any frustum corner inside the box (inclusive).  The kernels
    evaluate it as the AND over axes of 8-bit masks 'corners whose coordinate on this axis lies in [lo, hi]', built from the
    DISTINCT coordinates per axis (bit-pattern distinct: -0 and +0 stay separate entries)."""
    rng = np.random.default_rng(7)
    for trial in range(300):
        # frustum-like corner sets with many repeated coordinates, zeros of both signs included
        vals = np.array([-0.0, 0.0, -0.01, 0.01, -1.0, 1.0, -120.0, 120.0, 2.5], f32)
        corners = vals[rng.integers(0, len(vals), (8, 3))]
        m = 4000
        a = (rng.normal(size=(m, 3)) * 2).astype(f32)
        b = (rng.normal(size=(m, 3)) * 2).astype(f32)
        snap = rng.random((m, 3)) < 0.3  # box bounds that coincide with corner coordinates (inclusive compares matter)
        a = np.where(snap, vals[rng.integers(0, len(vals), (m, 3))], a)
        lo, hi = np.minimum(a, b), np.maximum(a, b)
        want = np.zeros(m, bool)
        for c in range(8):
            want |= ((corners[c] >= lo) & (corners[c] <= hi)).all(1)
        alive = np.full(m, 0xFF, np.uint32)
        for ax in range(3):
            bits = corners[:, ax].view(np.uint32)
            mask = np.zeros(m, np.uint32)
            for u in np.unique(bits):
                v = np.array([u], np.uint32).view(f32)[0]
                cm = np.uint32(sum(1 << i for i in range(8) if bits[i] == u))
                mask |= np.where((v >= lo[:, ax]) & (v <= hi[:, ax]), cm, np.uint32(0))
            alive &= mask
        assert np.array_equal(alive != 0, want), trial


def test_cube_face_frusta_share_planes_and_what_sharing_would_buy():
    """VERDICT r01 item 4(ii) asked whether plane evaluations can be shared between the frusta of one call.  Facts this test pins
    for the benchmark's six cube-face frusta (camera.cube_frusta): the 24 side planes are 6 unoriented planes — every side
    plane is bit-identical to a side plane of one other face and the negation (up to the sign of zero components) of the
    side planes of two more.  Sharing is exact: for the negated plane the reference's s is -(n·p) + d' (rounding is symmetric
    under negation), so "all corners behind" is  d' - min_corner(n·p) <= 0  with min_corner built per axis like the max-corner.
    The kernels do NOT use it: the per-frustum form tests a plane PAIR at a time with a warp-vote early exit after the first
    rejecting pair, which a shared form would lose."""
    from fyrox_b200 import camera
    fr = camera.cube_frusta()
    P = np.array([np.ctypeslib.as_array(f.planes) for f in fr], f32).reshape(36, 4)
    u32 = lambda v: np.ascontiguousarray(v, f32).view(np.uint32)
    canon = lambda v: np.where(v == 0, f32(0.0), v)  # +0 for both zeros
    ident = neg = 0
    for i in range(36):
        for j in range(i + 1, 36):
            if i // 6 == j // 6:
                continue
            ident += bool((u32(P[i]) == u32(P[j])).all())
            neg += bool((u32(canon(P[i][:3])) == u32(canon(-P[j][:3]))).all())
    assert ident == 12 and neg >= 24, (ident, neg)
    # exactness of the shared form on the negated plane, random + adversarial cases
    rng = np.random.default_rng(5)
    with np.errstate(over="ignore", under="ignore", invalid="ignore"):
        for mode in ("random", "scaled", "special"):
            n, d, lo, hi = make_cases(rng, 500_000, mode)
            want = literal_all_behind(-n, d, lo, hi)
            # min-corner of +n: operand picked the other way round
            vx = np.where(n[:, 0] < 0, hi[:, 0], lo[:, 0])
            vy = np.where(n[:, 1] < 0, hi[:, 1], lo[:, 1])
            vz = np.where(n[:, 2] < 0, hi[:, 2], lo[:, 2])
            s_min = (n[:, 0] * vx + n[:, 1] * vy) + n[:, 2] * vz
            got = (-s_min + d) <= 0
            assert np.array_equal(got, want), (mode, int((got != want).sum()))


def test_strong_reject_skips_the_corner_fallback_exactly():
    """frustum_intersects_aabb (fyx_math.cuh) skips the corner-in-box fallback of Frustum::is_intersects_aabb (frustum.rs:236-242)
    when, on some plane, the box's max-corner value s is BELOW pm = the smallest s over the frustum's own eight corners (computed
    by the host with the same operations).  Claim: then no frustum corner lies inside the box, so the fallback is false.  Checked
    on real frusta (their corners sit on the planes up to rounding: pm is a few ulps around zero — the touching cases are the
    point) and on arbitrary plane / corner sets, with boxes snapped onto corners and planes."""
    from fyrox_b200 import camera
    rng = np.random.default_rng(31)
    real = []
    for f in camera.cube_frusta((1.5, -2.0, 0.25), 300.0):
        real.append((np.ctypeslib.as_array(f.planes).astype(f32).reshape(6, 4), np.ctypeslib.as_array(f.corners).astype(f32).reshape(8, 3)))
    skipped = inside_total = weak = 0
    with np.errstate(over="ignore", under="ignore", invalid="ignore"):
        for trial in range(40):
            if trial < 24:
                P, corners = real[trial % 6]
                n, d = P[:, :3].copy(), P[:, 3].copy()
            elif trial < 32:
                n = rng.normal(size=(6, 3)).astype(f32)
                d = (rng.normal(size=6) * 30).astype(f32)
                corners = (rng.normal(size=(8, 3)) * 40).astype(f32)
            else:
                n = special_values(rng, 18).reshape(6, 3)
                d = special_values(rng, 6)
                corners = special_values(rng, 24).reshape(8, 3)
            m = 200_000
            # boxes: around the corners (tiny to large), some bounds exactly ON corner coordinates
            base = corners[rng.integers(0, 8, m)]
            ext = (10.0 ** rng.uniform(-7, 2, (m, 1))).astype(f32)
            a = base + (rng.normal(size=(m, 3)).astype(f32) * ext)
            b = base + (rng.normal(size=(m, 3)).astype(f32) * ext)
            snap = rng.random((m, 3)) < 0.25
            a = np.where(snap, corners[rng.integers(0, 8, m)], a)
            if trial >= 32:
                sv = special_values(rng, m * 3).reshape(m, 3)
                b = np.where(rng.random((m, 3)) < 0.4, sv, b)
            lo, hi = np.minimum(a, b), np.maximum(a, b)
            # pm per plane, same arithmetic
            pm = np.empty(6, f32)
            for p in range(6):
                sv_ = ((n[p, 0] * corners[:, 0] + n[p, 1] * corners[:, 1]) + n[p, 2] * corners[:, 2]) + d[p]
                pm[p] = np.nan if np.isnan(sv_).any() else sv_.min()
            strong = np.zeros(m, bool)
            rejected = np.zeros(m, bool)
            for p in range(6):
                npl = np.broadcast_to(n[p], (m, 3))
                vx = np.where(npl[:, 0] < 0, lo[:, 0], hi[:, 0])
                vy = np.where(npl[:, 1] < 0, lo[:, 1], hi[:, 1])
                vz = np.where(npl[:, 2] < 0, lo[:, 2], hi[:, 2])
                s = s_of(npl, np.full(m, d[p], f32), vx, vy, vz)
                strong |= s < pm[p]
                rejected |= s <= 0
            inside = np.zeros(m, bool)
            for c in range(8):
                inside |= ((corners[c] >= lo) & (corners[c] <= hi)).all(1)
            bad = strong & inside
            assert not bad.any(), (trial, int(bad.sum()), lo[bad][:2], hi[bad][:2])
            skipped += int((strong & rejected).sum())
            weak += int((rejected & ~strong).sum())
            inside_total += int(inside.sum())
    assert skipped > 100_000 and inside_total > 100_000 and weak > 1000, (skipped, inside_total, weak)
