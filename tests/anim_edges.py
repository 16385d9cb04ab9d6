"""Edge cases of the animation step (N2): curve sampling with span hints, time advance and pose blending, where a
restatement of fyrox-math/src/curve.rs, lib.rs and fyrox-animation/src/value.rs goes wrong.

Two restatements of the same operations, both written from the reference source (not from the oracle):

* the float32 form (`wrapf`, `stepf`, `lerpf`, `cubicf`, `key_interpolate`, `curve_value_at`, `quat_from_euler_xyz`,
  `track_value_blend`): numpy float32 scalars, one IEEE rounding per operation, no FMA, operations in the order Rust
  evaluates them.  sin / cos come from the platform libm, as Rust's f32::sin_cos does.  It must equal the oracle bit for
  bit, and the kernels must equal the oracle bit for bit (Euler tracks: to the libm tolerance).
* the float64 form (`*64`): the same formulas as mathematics, evaluated in float64 on the same float32 inputs.  The
  discrete choices (which branch of wrapf, which span of the curve, which key's kind picks the family) are made by
  exact comparisons of float32 inputs and are the same in both forms; only the arithmetic differs.

The float32 path must stay within these bounds of the float64 value (u = 2^-24, the float32 unit roundoff;
ulp(x) = the float32 spacing at |x|).  Each bound is rounding steps x term magnitude, with a margin of about two; the
largest ratio error / bound seen on the generated cases is printed by the CPU and GPU tests and recorded in DESIGN.md.

* lerp `a + (b - a) t`, t = (x - l) / (r - l): t carries three roundings (two subtractions, one division): |dt| <= 3u t.
  Then b - a, * t and + a round once each.  |err| <= 10u |b - a| + 2u max(|a|, |b|).   (LERP_A, LERP_B)
* cubic Hermite (curve.rs / lib.rs:212-221): four terms, each a basis polynomial of t (intermediates up to 3 in
  magnitude, about five roundings) times p0, p1 or m * scale; three additions.  With M = |p0| + |p1| +
  (|m0| + |m1|) |p1 - p0|: |err| <= 40u M.  The t error moves the value by at most |dv/dt| 3u <= 3u M.   (CUBIC_K)
  Skipped: curves whose float32 value or any term overflows (not finite in float32) - the float32 path is then
  inf / NaN and the float64 value is finite; the oracle comparison still covers them.
* step (Constant left key): exact, except where t rounds to 1 in float32 while t < 1 in float64 (`t_one` cases):
  stepf is discontinuous there, so the float64 check skips Constant spans with t64 >= 1 - 4u.
* wrapf as a float64 modulus: lo + ((n - lo) mod len), compared as a phase (distance modulo len), since a result
  one period away is the same time on a looped slice.  n - lo, num * len, the subtraction and + lo round once each, and
  len = hi - lo rounds once, an error multiplied by num: |err| <= 3 ulp(n - lo) + (num + 1) ulp(len) + 2 ulp(max(|lo|, |hi|)).
  Skipped: |n / len| >= 2^24 (the float32 quotient no longer resolves whole periods) and len = 0.   (wrap_bound)
* quat_from_euler -> rotation matrix with float64 sin / cos: the float32 sin / cos are within 2 ulp (libm <= 1, CUDA
  sincosf <= 2), each quaternion component is at most two products of three such factors and one sum, the rotation
  matrix entries (`1 - 2(y^2 + z^2)`, `2(xy - wz)`, ...) add about six roundings on terms bounded by 2:
  quaternion components |err| <= 16u, rotation-matrix entries |err| <= 48u.   (EULER_QUAT_BOUND, EULER_MAT_BOUND)
* TrackValue::blend_with: vectors `a (1 - w) + b w`: 1 - w, two products and a sum round once each:
  |err| <= 4u (|a| |1 - w| + |b| |w|).  Rotations: the same per component on unit inputs, then the short-way flip and
  normalisation by N = |o| (dot, sqrt and division: about four roundings): |err| <= 8u (|1 - w| + |w|) / N + 6u.
  Skipped: rotations whose float64 dot is within 8u of 0 with a non-zero value (the flip decision itself may differ).
"""
from __future__ import annotations

import ctypes as C
import ctypes.util
import math

import numpy as np

import oracle_binding as ob

f32 = np.float32
U = 2.0 ** -24
KD = ob.KEY_DTYPE
CONST, LIN, CUB = ob.KEY_CONSTANT, ob.KEY_LINEAR, ob.KEY_CUBIC

LERP_A, LERP_B = 10.0, 2.0
CUBIC_K = 40.0
EULER_QUAT_BOUND = 16 * U
EULER_MAT_BOUND = 48 * U

_libm = C.CDLL(ctypes.util.find_library("m"))
_libm.sinf.restype = _libm.cosf.restype = C.c_float
_libm.sinf.argtypes = _libm.cosf.argtypes = [C.c_float]


def same_bits(a, b) -> bool:
    """Bit equality of two float32 values; any NaN equals any NaN (helpers.bits_equal)."""
    a, b = np.array([a], np.float32), np.array([b], np.float32)
    return bool((a.view(np.uint32) == b.view(np.uint32))[0] or (np.isnan(a) & np.isnan(b))[0])


def ulp(x) -> float:
    return float(np.spacing(np.abs(f32(x))))


# ---- float32 restatement (fyrox-math/src/lib.rs, curve.rs; fyrox-animation/src/value.rs; nalgebra op orders) -------

def wrapf(n, lo, hi):
    """lib.rs:179-203."""
    n, lo, hi = f32(n), f32(lo), f32(hi)
    if n >= lo and n <= hi:
        return n
    if hi == 0 and lo == 0:
        return f32(0)
    hi = f32(hi - lo)
    offset = lo
    lo = f32(0)
    n = f32(n - offset)
    with np.errstate(all="ignore"):
        num_of_max = f32(np.floor(np.abs(f32(n / hi))))
        if n >= hi:
            n = f32(n - f32(num_of_max * hi))
        elif n < lo:
            n = f32(n + f32(f32(num_of_max + f32(1)) * hi))
        return f32(n + offset)


def stepf(p0, p1, t):
    """curve.rs:25-31."""
    return f32(p1) if f32(t) == f32(1) else f32(p0)


def lerpf(a, b, t):
    """lib.rs:206-208."""
    return f32(f32(a) + f32(f32(f32(b) - f32(a)) * f32(t)))


def cubicf(p0, p1, t, m0, m1):
    """lib.rs:212-221: sums and products left to right."""
    p0, p1, t, m0, m1 = f32(p0), f32(p1), f32(t), f32(m0), f32(m1)
    with np.errstate(all="ignore"):
        t2 = f32(t * t)
        t3 = f32(t2 * t)
        scale = f32(abs(f32(p1 - p0)))
        a = f32(f32(f32(f32(f32(2) * t3) - f32(f32(3) * t2)) + f32(1)) * p0)
        b = f32(f32(f32(f32(f32(t3 - f32(f32(2) * t2)) + t) * m0)) * scale)
        c = f32(f32(f32(f32(-2) * t3) + f32(f32(3) * t2)) * p1)
        d = f32(f32(f32(f32(t3 - t2) * m1)) * scale)
        return f32(f32(f32(a + b) + c) + d)


def key_interpolate(l, r, t):
    """interpolate (curve.rs:87-133): the LEFT key's kind picks the family; a cubic pairs the left key's right tangent
    with the right key's left tangent if the right key is cubic too, else with 0.  Keys are KEY_DTYPE records."""
    if int(l["kind"]) == CONST:
        return stepf(l["value"], r["value"], t)
    if int(l["kind"]) == LIN:
        return lerpf(l["value"], r["value"], t)
    m1 = r["left_tangent"] if int(r["kind"]) == CUB else 0.0
    return cubicf(l["value"], r["value"], t, l["right_tangent"], m1)


def span_t(l, r, x):
    with np.errstate(all="ignore"):
        return f32(f32(f32(x) - f32(l["location"])) / f32(f32(r["location"]) - f32(l["location"])))


def find_span(keys, x, hint):
    """Curve::fetch_at's span choice (curve.rs:272-305), exact comparisons only.  Returns ("first" | "last" | "hint" |
    "search", left index, right index, new hint)."""
    n = len(keys)
    x = f32(x)
    loc = keys["location"]
    if x <= loc[0]:
        return "first", 0, 0, 0
    if x >= loc[n - 1]:
        return "last", n - 1, n - 1, n - 1
    li = max(hint - 1, 0)
    if li < n and hint < n and loc[li] <= x < loc[hint]:
        return "hint", li, hint, hint
    lo = int(np.searchsorted(loc, x, side="left"))  # partition_point(|k| k.location < x)
    return "search", max(lo - 1, 0), lo, lo


def curve_value_at(keys, x, hint=0):
    """Curve::value_at = fetch_at with CurveKey::interpolate (curve.rs:252-314).  Returns (value, new hint)."""
    if len(keys) == 0:
        return f32(0), hint
    how, li, ri, h = find_span(keys, x, hint)
    if how in ("first", "last"):
        return f32(keys[li]["value"]), h
    return key_interpolate(keys[li], keys[ri], span_t(keys[li], keys[ri], x)), h


def _quat_mul(a, b):
    """nalgebra quaternion product, components (i, j, k, w), the oracle header's op order."""
    w = f32(f32(f32(f32(a[3] * b[3]) - f32(a[0] * b[0])) - f32(a[1] * b[1])) - f32(a[2] * b[2]))
    i = f32(f32(f32(f32(a[3] * b[0]) + f32(a[0] * b[3])) + f32(a[1] * b[2])) - f32(a[2] * b[1]))
    j = f32(f32(f32(f32(a[3] * b[1]) - f32(a[0] * b[2])) + f32(a[1] * b[3])) + f32(a[2] * b[0]))
    k = f32(f32(f32(f32(a[3] * b[2]) + f32(a[0] * b[1])) - f32(a[1] * b[0])) + f32(a[2] * b[3]))
    return [i, j, k, w]


def quat_from_euler_xyz(e):
    """quat_from_euler(v, RotationOrder::XYZ) = qz * qy * qx (lib.rs:725-740), from_axis_angle = (axis * sin, cos) of
    angle / 2."""
    q = []
    for a in range(3):
        h = f32(f32(e[a]) / f32(2))
        s, c = f32(_libm.sinf(h)), f32(_libm.cosf(h))
        q.append([f32(f32(1.0 if b == a else 0.0) * s) for b in range(3)] + [c])
    return np.array(_quat_mul(_quat_mul(q[2], q[1]), q[0]), np.float32)


def _dot4(a, b):
    return f32(f32(f32(a[0] * b[0]) + f32(a[2] * b[2])) + f32(f32(a[1] * b[1]) + f32(a[3] * b[3])))


def track_value_blend(is_quat, a, b, w):
    """TrackValue::blend_with (value.rs:201-227): nalgebra lerp a*(1-w) + b*w; rotations take the short way
    (value.rs:449-454) and are re-normalised (q_i / sqrt(dot4(q, q)))."""
    a, b, w = np.asarray(a, np.float32), np.asarray(b, np.float32), f32(w)
    u = f32(f32(1) - w)
    s = a.copy()
    with np.errstate(all="ignore"):
        if is_quat and _dot4(s, b) < 0:
            s = -s
        o = np.array([f32(f32(s[i] * u) + f32(b[i] * w)) for i in range(4)], np.float32)
        if is_quat:
            n = f32(np.sqrt(_dot4(o, o)))
            o = np.array([f32(o[i] / n) for i in range(4)], np.float32)
    return o


# ---- float64 reference -------------------------------------------------------------------------------------------

def key_interpolate64(l, r, t64):
    """The same family choice, the formulas in float64 at a float64 t."""
    p0, p1 = float(l["value"]), float(r["value"])
    if int(l["kind"]) == CONST:
        return p1 if t64 == 1.0 else p0
    if int(l["kind"]) == LIN:
        return p0 + (p1 - p0) * t64
    m0 = float(l["right_tangent"])
    m1 = float(r["left_tangent"]) if int(r["kind"]) == CUB else 0.0
    t2, t3 = t64 * t64, t64 ** 3
    s = abs(p1 - p0)
    return (2 * t3 - 3 * t2 + 1) * p0 + (t3 - 2 * t2 + t64) * m0 * s + (-2 * t3 + 3 * t2) * p1 + (t3 - t2) * m1 * s


def curve_value_at64(keys, x, hint=0):
    """Returns (float64 value, bound on |float32 - float64|, or None when the case is skipped)."""
    if len(keys) == 0:
        return 0.0, 0.0
    how, li, ri, _ = find_span(keys, x, hint)
    if how in ("first", "last"):
        return float(keys[li]["value"]), 0.0
    l, r = keys[li], keys[ri]
    t64 = (float(f32(x)) - float(l["location"])) / (float(r["location"]) - float(l["location"]))
    v = key_interpolate64(l, r, t64)
    p0, p1 = float(l["value"]), float(r["value"])
    kind = int(l["kind"])
    if kind == CONST:
        return v, (None if t64 >= 1 - 4 * U else 0.0)
    if kind == LIN:
        return v, LERP_A * U * abs(p1 - p0) + LERP_B * U * max(abs(p0), abs(p1))
    m0 = float(l["right_tangent"])
    m1 = float(r["left_tangent"]) if int(r["kind"]) == CUB else 0.0
    M = abs(p0) + abs(p1) + (abs(m0) + abs(m1)) * abs(p1 - p0)
    if not (M < 1e37 and np.isfinite(key_interpolate(l, r, span_t(l, r, x)))):
        return v, None  # the float32 terms overflow: skipped
    return v, CUBIC_K * U * M


def wrapf64(n, lo, hi):
    """wrapf as mathematics on the float32 inputs: n itself inside [lo, hi], the (0, 0) short-cut, else
    lo + ((n - lo) mod len)."""
    n, lo, hi = float(f32(n)), float(f32(lo)), float(f32(hi))
    if lo <= n <= hi:
        return n
    if hi == 0 and lo == 0:
        return 0.0
    return lo + math.fmod(math.fmod(n - lo, hi - lo) + (hi - lo), hi - lo)


def wrap_bound(n, lo, hi):
    """Bound on the phase distance of wrapf from wrapf64, None when skipped (see the module docstring)."""
    n, lo, hi = float(f32(n)), float(f32(lo)), float(f32(hi))
    if lo <= n <= hi or (hi == 0 and lo == 0):
        return 0.0
    ln = hi - lo
    if ln == 0 or abs((n - lo) / ln) >= 2.0 ** 24:
        return None
    num = math.floor(abs((n - lo) / ln))
    return 3 * ulp(n - lo) + (num + 1) * ulp(ln) + 2 * ulp(max(abs(lo), abs(hi)))


def phase_distance(a, b, lo, hi):
    ln = float(f32(hi)) - float(f32(lo))
    d = abs(float(a) - float(b))
    return d if ln <= 0 else min(d % ln, ln - d % ln)


def quat_from_euler64(e):
    def axis(k, ang):
        q = [0.0, 0.0, 0.0, math.cos(ang / 2)]
        q[k] = math.sin(ang / 2)
        return q

    def mul(a, b):
        return [a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1],
                a[3] * b[1] - a[0] * b[2] + a[1] * b[3] + a[2] * b[0],
                a[3] * b[2] + a[0] * b[1] - a[1] * b[0] + a[2] * b[3],
                a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2]]

    e = [float(f32(v)) for v in e]
    return np.array(mul(mul(axis(2, e[2]), axis(1, e[1])), axis(0, e[0])))


def rotation_matrix64(q):
    """Column-major 3x3 (as the 16-float matrices store it: m[0..2] = first column) of a unit quaternion (i, j, k, w)."""
    x, y, z, w = q
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                  [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                  [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])
    return R.T.reshape(9)


def track_value_blend64(is_quat, a, b, w):
    """Returns (float64 value, bound, or None when the short-way decision is within rounding of 0)."""
    a, b, w = np.asarray(a, np.float64), np.asarray(b, np.float64), float(f32(w))
    if not is_quat:
        return a * (1 - w) + b * w, 4 * U * (np.abs(a) * abs(1 - w) + np.abs(b) * abs(w))
    d = float(a @ b)
    if d != 0 and abs(d) <= 8 * U:
        return None, None
    s = -a if d < 0 else a
    o = s * (1 - w) + b * w
    N = float(np.linalg.norm(o))
    return o / N, np.full(4, 8 * U * (abs(1 - w) + abs(w)) / N + 6 * U)


# ---- generators -----------------------------------------------------------------------------------------------------

def keys_of(rows):
    """rows of (location, value, kind, left_tangent, right_tangent) -> KEY_DTYPE, in the order given (sorted callers)."""
    k = np.zeros(len(rows), KD)
    for i, r in enumerate(rows):
        k[i] = tuple(r) + (0.0,) * (5 - len(r))
    return k


def random_curve(rng, n, lo_loc=-3.0, hi_loc=3.0, kinds=(CONST, LIN, CUB), vmax=3.0, tmax=1.5, dups=False):
    locs = np.sort(rng.uniform(lo_loc, hi_loc, n).astype(np.float32))
    if dups and n > 3:
        locs[rng.integers(1, n - 1)] = locs[rng.integers(0, n)]
        locs = np.sort(locs)
    kinds = rng.choice(kinds, n)
    return keys_of([(locs[i], f32(rng.uniform(-vmax, vmax)), int(kinds[i]), f32(rng.uniform(-tmax, tmax)),
                     f32(rng.uniform(-tmax, tmax))) for i in range(n)])


def nearest_t_one(l_loc, r_loc):
    """The largest float32 x < r_loc with (x - l) / (r - l) == 1.0 in float32, or None."""
    l_loc, r_loc = f32(l_loc), f32(r_loc)
    x = np.nextafter(r_loc, f32(-np.inf))
    best = None
    for _ in range(64):
        if x <= l_loc:
            break
        if span_t({"location": l_loc}, {"location": r_loc}, x) == f32(1):
            best = x
        else:
            break
        x = np.nextafter(x, f32(-np.inf))
    return best


CURVE_CLASSES = ("on_key", "key_ulp_below", "key_ulp_above", "first_last", "first_last_ulp_inside", "t_one",
                 "duplicates_start", "duplicates_middle", "duplicates_end", "span_one_ulp", "large_locations",
                 "kind_pairs", "overflow", "key_counts")


def curve_cases(rng):
    """{class: [(keys, [location, ...]), ...]}: each curve with the probe locations that make it that class.  Probes are
    sampled with hint 0 and with every hint (hint_cases covers the hint sequences)."""
    out = {c: [] for c in CURVE_CLASSES}
    dn = lambda x: np.nextafter(f32(x), f32(-np.inf))
    up = lambda x: np.nextafter(f32(x), f32(np.inf))
    for _ in range(12):
        k = random_curve(rng, 7)
        inner = k["location"][1:-1]
        out["on_key"].append((k, list(inner)))
        out["key_ulp_below"].append((k, [dn(x) for x in inner]))
        out["key_ulp_above"].append((k, [up(x) for x in inner]))
        out["first_last"].append((k, [k["location"][0], k["location"][-1], dn(k["location"][0]), up(k["location"][-1])]))
        out["first_last_ulp_inside"].append((k, [up(k["location"][0]), dn(k["location"][-1])]))
    # t == 1.0 although loc < r.loc: |l| much larger than |r|, so x - l rounds up to r - l
    while len(out["t_one"]) < 24:
        l = f32(-rng.uniform(10.0, 3000.0))
        r = f32(rng.uniform(0.001, 2.0))
        x = nearest_t_one(l, r)
        if x is None or x >= r:
            continue
        kinds = [(CONST, LIN), (LIN, CUB), (CUB, CUB), (CONST, CONST)][len(out["t_one"]) % 4]
        k = keys_of([(f32(l - 1), 0.5, LIN), (l, f32(rng.uniform(-3, 3)), kinds[0], 0.7, -0.4),
                     (r, f32(rng.uniform(-3, 3)), kinds[1], 1.3, 0.2), (f32(r + 1), 0.25, LIN)])
        out["t_one"].append((k, [x]))
    for cls, m_at in (("duplicates_start", lambda m: slice(0, m)), ("duplicates_middle", lambda m: slice(3, 3 + m)),
                      ("duplicates_end", lambda m: slice(7 - m, 7))):
        for m in (2, 3):
            for _ in range(3):
                k = random_curve(rng, 7)
                sl = m_at(m)
                d = k["location"][sl.start] if cls != "duplicates_end" else k["location"][6]
                k["location"][sl] = d
                out[cls].append((k, [d, dn(d), up(d), k["location"][0], k["location"][-1]]))
    for _ in range(12):
        a = f32(rng.uniform(-100, 100))
        b = up(a)
        k = keys_of([(f32(a - 1), 1.0, LIN), (a, f32(rng.uniform(-3, 3)), int(rng.integers(0, 3)), 0.5, -2.0),
                     (b, f32(rng.uniform(-3, 3)), int(rng.integers(0, 3)), 1.0, 1.0), (f32(b + 1), 0.0, LIN)])
        out["span_one_ulp"].append((k, [a, b]))
    for mag in (1e4, 1e5, 1e6):
        for _ in range(4):
            k = random_curve(rng, 9, mag, mag * 1.05)
            probes = list(rng.uniform(mag, mag * 1.05, 12).astype(np.float32)) + [dn(x) for x in k["location"][1:-1]]
            out["large_locations"].append((k, probes))
    for lk in (CONST, LIN, CUB):
        for rk in (CONST, LIN, CUB):
            for _ in range(2):
                k = keys_of([(0.0, f32(rng.uniform(-3, 3)), lk, f32(rng.uniform(-2, 2)), f32(rng.uniform(-2, 2))),
                             (1.0, f32(rng.uniform(-3, 3)), rk, f32(rng.uniform(-2, 2)), f32(rng.uniform(-2, 2)))])
                out["kind_pairs"].append((k, list(np.linspace(0.05, 0.95, 7).astype(np.float32)) + [dn(1.0)]))
    for i in range(10):
        big = f32(10.0 ** rng.uniform(20, 30)) if i % 2 else f32(rng.uniform(1e38, 3e38))  # |p1 - p0| overflows
        tan = f32(10.0 ** rng.uniform(3, 7)) * f32(rng.choice([-1, 1]))
        k = keys_of([(0.0, big * f32(rng.choice([-1, 1])), CUB, tan, tan), (1.0, -big, CUB, -tan, tan),
                     (2.0, big, CUB, tan, -tan)])
        out["overflow"].append((k, list(np.linspace(0.1, 1.9, 9).astype(np.float32))))
    for n in (0, 1, 2, 3, 31, 32, 33, 1000, 70000):
        k = random_curve(rng, n, -3.0, 3.0) if n else keys_of([])
        probes = list(rng.uniform(-3.2, 3.2, 16).astype(np.float32))
        if n:
            probes += [k["location"][n // 2], dn(k["location"][n // 2]), k["location"][-1], k["location"][0]]
        out["key_counts"].append((k, probes))
    return out


HINT_CLASSES = ("forward", "backward", "wrap_jump", "key_after_left_span", "key_after_right_span")


def lerp_one_differs(a, b):
    return lerpf(a, b, 1.0) != f32(b)


def hint_cases(rng):
    """{class: [(keys, [time, ...]), ...]}: a curve and the times it is sampled at in order, the hint carried along."""
    out = {c: [] for c in HINT_CLASSES}
    for _ in range(8):
        k = random_curve(rng, int(rng.integers(6, 40)), 0.0, 4.0)
        out["forward"].append((k, list(np.sort(rng.uniform(-0.2, 4.2, 24)).astype(np.float32))))
        k = random_curve(rng, int(rng.integers(6, 40)), 0.0, 4.0)
        out["backward"].append((k, list(np.sort(rng.uniform(-0.2, 4.2, 24))[::-1].astype(np.float32))))
        k = random_curve(rng, int(rng.integers(6, 40)), 0.0, 4.0)
        ts = np.concatenate([np.linspace(2.5, 3.9, 6), np.linspace(0.1, 1.5, 6), np.linspace(3.0, 3.9, 4), [0.05]])
        out["wrap_jump"].append((k, list(ts.astype(np.float32))))
    # a key whose two evaluations differ: lerp(a, b, 1) != b on the left span, exactly b on the right span
    while len(out["key_after_left_span"]) < 16:
        k = random_curve(rng, 8, 0.0, 4.0, kinds=(LIN,), vmax=1.0)
        j = int(rng.integers(2, 6))
        if not lerp_one_differs(k["value"][j - 1], k["value"][j]) or len(np.unique(k["location"])) < 8:
            continue
        xj = k["location"][j]
        left = f32((k["location"][j - 1] + xj) / 2)
        right = f32((xj + k["location"][j + 1]) / 2)
        out["key_after_left_span"].append((k, [left, xj, right, xj]))
        out["key_after_right_span"].append((k, [right, xj, left, xj]))
    return out


TIME_SLICES = {"inexact": (0.1, 0.7), "thirds": (-1 / 3, 5 / 7), "unit": (0.0, 2.0), "zero": (0.0, 0.0),
               "point": (1.25, 1.25), "large": (1000.1, 1003.7)}
TIME_CLASSES = ("inside", "on_end", "end_ulp_below", "end_ulp_above", "on_start_plus_k_len", "q_2_20", "q_2_23",
                "q_2_24", "negative", "speed_zero", "speed_negative", "speed_1e6", "dt_zero")


K_LENS = (2, 3, 7, -1, -2, -5)


def speed_for(t0, target):
    """A float32 speed s with fl(t0 + s) == target (dt = 1), or None."""
    t0, target = f32(t0), f32(target)
    s = f32(target - t0)
    for _ in range(8):
        got = f32(t0 + s)
        if got == target:
            return s
        s = np.nextafter(s, f32(np.inf) if got < target else f32(-np.inf))
    return None


def time_cases():
    """[(class, slice name, (lo, hi), looped, t0, speed)]: one animation each, ticked with dt = 1 (n = t0 + speed), then
    more ticks; `dt_zero` animations are ticked with dt = 0 first.  The float32 n each reaches on its first tick is
    `first_n`."""
    out = []
    for name, (lo, hi) in TIME_SLICES.items():
        lo, hi = f32(lo), f32(hi)
        ln = f32(hi - lo)
        t0 = lo
        for looped in (True, False):
            def add(cls, target=None, speed=None, start=t0):
                s = speed if speed is not None else speed_for(start, target)
                if s is not None:
                    out.append((cls, name, (lo, hi), looped, f32(start), f32(s)))
            add("inside", f32(lo + ln * f32(0.5)))
            add("on_end", hi)
            add("end_ulp_below", np.nextafter(hi, f32(-np.inf)))
            add("end_ulp_above", np.nextafter(hi, f32(np.inf)))
            for kk in K_LENS:
                add("on_start_plus_k_len", f32(lo + f32(f32(kk) * ln)))
            base = max(float(ln), 1e-3)
            for cls, q in (("q_2_20", 2 ** 20), ("q_2_23", 2 ** 23), ("q_2_24", 2 ** 24)):
                for sgn in (1, -1):
                    for j in (-1, 0, 1):
                        add(cls, f32(lo + sgn * (q + j) * base + sgn * 0.37 * base))
            for tgt in (-0.3, -7.9, -1e3, -abs(float(lo)) - 3.5 * float(ln) - 1.0):
                add("negative", f32(tgt))
            add("speed_zero", speed=0.0)
            add("speed_negative", speed=-0.55)
            add("speed_negative", speed=-13.0)
            add("speed_1e6", speed=1e6)
            add("speed_1e6", speed=-1e6)
            add("dt_zero", speed=0.9)
    return out


def first_n(case):
    _, _, _, _, t0, s = case
    return f32(t0 + f32(f32(1) * s))


EULER_CLASSES = ("small", "near_half_pi", "around_1e3", "around_1e5", "around_1e6")


def euler_cases(rng):
    """{class: [angles (3,) float32, ...]}."""
    out = {c: [] for c in EULER_CLASSES}
    for _ in range(48):
        out["small"].append(rng.uniform(-4, 4, 3).astype(np.float32))
        k = rng.integers(-8, 9, 3)
        out["near_half_pi"].append((k * (np.pi / 2) + rng.choice([0.0, 1e-7, -1e-7, 1e-3], 3)).astype(np.float32))
        for cls, mag in (("around_1e3", 1e3), ("around_1e5", 1e5), ("around_1e6", 1e6)):
            out[cls].append((rng.choice([-1, 1], 3) * rng.uniform(0.9, 1.1, 3) * mag).astype(np.float32))
    return out


BLEND_CLASSES = ("weights", "antipodal", "dot_plus_zero", "dot_minus_zero", "random_quat", "vectors")
BLEND_WEIGHTS = (0.0, 1.0, -0.5, 2.0, 0.3)


def unit_quat(rng):
    q = rng.normal(size=4).astype(np.float32)
    return (q / np.linalg.norm(q)).astype(np.float32)


def blend_cases(rng):
    """{class: [(is_quat, a (4,), b (4,), w), ...]} for TrackValue::blend_with."""
    out = {c: [] for c in BLEND_CLASSES}
    for w in BLEND_WEIGHTS:
        for _ in range(6):
            out["weights"].append((True, unit_quat(rng), unit_quat(rng), f32(w)))
            out["vectors"].append((False, np.r_[rng.uniform(-9, 9, 3), 0].astype(np.float32),
                                   np.r_[rng.uniform(-9, 9, 3), 0].astype(np.float32), f32(w)))
        for _ in range(4):
            a = unit_quat(rng)
            out["antipodal"].append((True, a, (-a).astype(np.float32), f32(w)))
        # dot4 = (a0*b0 + a2*b2) + (a1*b1 + a3*b3) exactly +0 / -0: products of zeros with signs chosen
        out["dot_plus_zero"].append((True, np.array([1, 0, 0, 0], np.float32), np.array([0, 1, 0, 0], np.float32), f32(w)))
        out["dot_plus_zero"].append((True, np.array([0.6, 0, 0.8, 0], np.float32), np.array([0, 0.8, 0, -0.6], np.float32), f32(w)))
        out["dot_minus_zero"].append((True, np.array([-0.0, 1, -0.0, 0], np.float32), np.array([1, -0.0, 1, -0.0], np.float32) / f32(np.sqrt(2)), f32(w)))
        out["dot_minus_zero"].append((True, np.array([1, -0.0, -0.0, -0.0], np.float32), np.array([-0.0, 1, 0, 1], np.float32) / f32(np.sqrt(2)), f32(w)))
    for _ in range(40):
        out["random_quat"].append((True, unit_quat(rng), unit_quat(rng), f32(rng.uniform(-0.5, 2.0))))
    return out


def zero_scale_pair():
    """A node driven by a player (scale x = +0) and then by a machine (scale x = -0) in one frame, under a parent whose
    translation is negative, so the sign of the zero survives into the node's global matrix."""
    def scale_anim(x):
        keys = keys_of([(0.0, x, CONST), (0.0, 1.0, CONST), (0.0, 1.0, CONST)])
        t = np.zeros(1, ob.TRACK_DTYPE)
        t[0]["target_node"], t[0]["binding"], t[0]["value_kind"], t[0]["enabled"], t[0]["n_curves"] = 2, ob.BIND_SCALE, ob.TV_VECTOR3, 1, 3
        t[0]["first_key"][:3] = [0, 1, 2]
        t[0]["n_keys"][:3] = [1, 1, 1]
        return t, keys
    parent = np.array([0xFFFFFFFF, 0, 1], np.uint32)
    trs = np.zeros((3, 10), np.float32)
    trs[:, 6] = trs[:, 7:10] = 1.0
    trs[1, 0:3] = -1.0
    return parent, trs, scale_anim(0.0), scale_anim(-0.0)


# ---- the oracle on the same inputs -------------------------------------------------------------------------------

def oracle_transforms(trs):
    """The oracle's Transform per node from (n, 10) position / rotation / scale rows."""
    arr = (ob.Transform * len(trs))()
    for i, t in enumerate(arr):
        ob.lib().orc_transform_identity(C.byref(t))
        t.local_position[:] = trs[i, 0:3].tolist()
        t.local_rotation[:] = trs[i, 3:7].tolist()
        t.local_scale[:] = trs[i, 7:10].tolist()
    return arr


def oracle_key_interpolate(l, r, t):
    kl = ob.CurveKey(float(l["location"]), float(l["value"]), int(l["kind"]), float(l["left_tangent"]), float(l["right_tangent"]))
    kr = ob.CurveKey(float(r["location"]), float(r["value"]), int(r["kind"]), float(r["left_tangent"]), float(r["right_tangent"]))
    return f32(ob.lib().orc_key_interpolate(C.byref(kl), C.byref(kr), float(t)))


def oracle_quat_from_euler(e):
    out = np.empty(4, np.float32)
    ob.lib().orc_quat_from_euler_xyz(ob.fp(np.ascontiguousarray(e, np.float32)), ob.fp(out))
    return out


def oracle_blend(is_quat, a, b, w):
    a = np.array(a, np.float32)
    ob.lib().orc_track_value_blend(int(is_quat), ob.fp(a), ob.fp(np.ascontiguousarray(b, np.float32)), float(w))
    return a
