"""Boxes on the rounding edge of Frustum::is_intersects_aabb (fyrox-math/src/frustum.rs:205-245), and the literal 8 corners x 6
planes loop to hold every device frustum-box test to.

The kernels do not run the reference's loop (fyx_math.cuh, frustum_intersects_aabb): they test one max corner per plane, reject
early against pm (the smallest plane value over the frustum's own corners, to_dev_frustum), evaluate the corner-in-box fallback
through masks of DISTINCT corner coordinates (a second half when an axis has more than four), and send non-tame boxes (huge,
non-finite, inverted) down a literal path lane by lane.  Each shortcut is exact only up to the last bit, so the boxes here sit
exactly where a bit decides:

  plane_zero / plane_above / plane_below   the max-corner value s of one plane is exactly 0, or the nearest value on either
                                            side of 0 that one-ulp steps of a box bound reach
  pm_equal / pm_below                      s equals pm, or is the nearest reachable value below it
  corner_on / corner_in / corner_out       the bounds picked by a plane's max corner lie exactly on a frustum corner, or one ulp
                                            beyond it (corner strictly inside) or short of it (corner outside)
  single_corner                            boxes that hold exactly one frustum corner
  point_plane / point_corner               zero-extent boxes on a plane (s == 0) and on each corner
  non_tame                                 |bound| > 1e18, +-inf, NaN, inverted

Everything is float32 with one rounding per operation, in the reference's order: s = ((nx*px + ny*py) + nz*pz) + d."""
from __future__ import annotations

import ctypes as C

import numpy as np

import oracle_binding as ob
from test_cull_trick_cpu import literal_all_behind, s_of, trick_all_behind

f32 = np.float32
KBIG = f32(1e18)  # aabb_is_tame's bound
# corners of each plane (frustum.rs:70-79: corner k = intersection of (L|R, T|B, F|N); planes L R T B F N)
FACE_CORNERS = ((0, 1, 4, 5), (2, 3, 6, 7), (0, 3, 4, 7), (1, 2, 5, 6), (0, 1, 2, 3), (4, 5, 6, 7))
CLASSES = ("plane_zero", "plane_above", "plane_below", "pm_equal", "pm_below", "corner_on", "corner_in", "corner_out", "single_corner",
           "point_plane", "point_corner", "non_tame")


def _boxes(boxes):
    b = np.ascontiguousarray(boxes, f32).reshape(-1, 6)
    return b[:, :3], b[:, 3:]


def literal_intersects(planes, corners, boxes):
    """Frustum::is_intersects_aabb, literally: outside iff for some plane all 8 box corners have s <= 0, else inside iff no such
    plane, or some frustum corner lies in the box (inclusive compares).  planes (6, 4), corners (8, 3), boxes (m, 6) as
    (min xyz, max xyz).  Returns (m,) bool."""
    P, Cn = np.asarray(planes, f32).reshape(6, 4), np.asarray(corners, f32).reshape(8, 3)
    lo, hi = _boxes(boxes)
    m = len(lo)
    cloud = np.ones(m, bool)
    with np.errstate(all="ignore"):
        for p in range(6):
            cloud &= ~literal_all_behind(np.broadcast_to(P[p, :3], (m, 3)), np.full(m, P[p, 3], f32), lo, hi)
        inside = np.zeros(m, bool)
        for c in range(8):
            inside |= ((Cn[c] >= lo) & (Cn[c] <= hi)).all(1)
    return cloud | inside


def dev_frustum_pm(planes, corners):
    """to_dev_frustum's pm: per plane the smallest s over the frustum's own corners, NaN if any of them is NaN."""
    P, Cn = np.asarray(planes, f32).reshape(6, 4), np.asarray(corners, f32).reshape(8, 3)
    with np.errstate(all="ignore"):
        s = s_of(np.broadcast_to(P[None, :, :3], (8, 6, 3)).reshape(48, 3), np.tile(P[:, 3], 8), np.repeat(Cn[:, 0], 6),
                 np.repeat(Cn[:, 1], 6), np.repeat(Cn[:, 2], 6)).reshape(8, 6)
    return np.where(np.isnan(s).any(0), f32(np.nan), np.nanmin(np.where(np.isnan(s), np.inf, s), 0)).astype(f32)


def is_tame(boxes):
    lo, hi = _boxes(boxes)
    with np.errstate(invalid="ignore"):
        return (np.abs(lo) <= KBIG).all(1) & (np.abs(hi) <= KBIG).all(1) & (lo <= hi).all(1)


def max_corner_s(planes, boxes):
    """(m, 6) s of each plane's max corner, the operand picked by the sign of the normal component as the kernels do."""
    P = np.asarray(planes, f32).reshape(6, 4)
    lo, hi = _boxes(boxes)
    m = len(lo)
    out = np.empty((m, 6), f32)
    with np.errstate(all="ignore"):
        for p in range(6):
            n = P[p, :3]
            v = [np.where(n[k] < 0, lo[:, k], hi[:, k]) for k in range(3)]
            out[:, p] = s_of(np.broadcast_to(n, (m, 3)), np.full(m, P[p, 3], f32), *v)
    return out


def _slack(planes, boxes):
    """(m, 6): a few ulps of the largest term of each plane's max-corner sum — the width of 'next to' a plane value."""
    P = np.asarray(planes, f32).reshape(6, 4)
    lo, hi = _boxes(boxes)
    with np.errstate(all="ignore"):
        big = np.abs(P[None, :, 3]) + 0 * lo[:, :1]
        for k in range(3):
            v = np.where(P[None, :, k] < 0, lo[:, k:k + 1], hi[:, k:k + 1])
            big = np.fmax(big, np.abs(P[None, :, k] * v))
        return f32(4) * np.spacing(big.astype(f32))


def classify(planes, corners, boxes):
    """Label -> (m,) bool of the world boxes, for the census: which edges of the predicate each decision stood on."""
    P, Cn = np.asarray(planes, f32).reshape(6, 4), np.asarray(corners, f32).reshape(8, 3)
    lo, hi = _boxes(boxes)
    tame = is_tame(boxes)
    s = max_corner_s(P, boxes)
    sl = _slack(P, boxes)
    pm = dev_frustum_pm(P, Cn)
    with np.errstate(all="ignore"):
        inside = np.stack([((Cn[c] >= lo) & (Cn[c] <= hi)).all(1) for c in range(8)], 1)
        on = np.zeros(len(lo), bool)
        ulp = np.zeros(len(lo), bool)
        for k in range(3):
            cv = Cn[:, k][None, :]
            for b in (lo[:, k:k + 1], hi[:, k:k + 1]):
                on |= (b.view(np.uint32) == cv.view(np.uint32)).any(1) & np.isfinite(b[:, 0])
                ulp |= ((np.nextafter(b, f32(np.inf)) == cv) | (np.nextafter(b, f32(-np.inf)) == cv)).any(1) & (b != cv).all(1)
        point = (lo == hi).all(1)
        lab = {
            "plane_zero": tame & (s == 0).any(1),
            "plane_above": tame & ((s > 0) & (s <= sl)).any(1),
            "plane_below": tame & ((s < 0) & (s >= -sl)).any(1),
            "pm_equal": tame & (s == pm[None]).any(1),
            "pm_below": tame & ((s < pm[None]) & (s >= pm[None] - sl)).any(1),
            "corner_on": tame & on & ~point,
            "corner_in": tame & ulp & inside.any(1) & ~point,
            "corner_out": tame & ulp & ~inside.any(1) & ~point,
            "single_corner": tame & (inside.sum(1) == 1) & ~point,
            "point_plane": tame & point & (s == 0).any(1) & ~inside.any(1),
            "point_corner": tame & point & inside.any(1),
            "non_tame": ~tame,
        }
        # the decisions only the corner-in-box fallback takes: every plane's cloud test fails and no strong reject fires
        cloud = ~np.stack([(s[:, p] <= 0) for p in range(6)], 1).any(1)
        strong = (s < pm[None]).any(1)
        lab["fallback"] = tame & ~cloud & ~strong
        lab["fallback_true"] = lab["fallback"] & inside.any(1)
        # ... and of those, the ones a corner decides whose coordinate is entry 4..7 of an axis's distinct list (n_ax > 4)
        hi_half = np.zeros(len(lo), bool)
        for k in range(3):
            _, first = np.unique(Cn[:, k].view(np.uint32), return_index=True)
            order = np.sort(first)
            if len(order) > 4:
                late = np.isin(Cn[:, k].view(np.uint32), Cn[order[4:], k].view(np.uint32))
                hi_half |= (inside & late[None]).any(1)
        lab["fallback_late_coord"] = lab["fallback_true"] & hi_half
    return lab


# ---- the kernels' form, in numpy ---------------------------------------------------------------------------------------------
def kernel_intersects(planes, corners, boxes):
    """frustum_intersects_aabb restated: tame boxes take the max corner per plane (trick_all_behind) and the pm reject, the rest
    the literal loop; then the fallback over DISTINCT corner coordinates per axis (bit-pattern distinct, unused entries NaN),
    the second half of each list only where that axis has more than four."""
    P, Cn = np.asarray(planes, f32).reshape(6, 4), np.asarray(corners, f32).reshape(8, 3)
    lo, hi = _boxes(boxes)
    m = len(lo)
    tame = is_tame(boxes)
    pm = dev_frustum_pm(P, Cn)
    cloud = np.ones(m, bool)
    with np.errstate(all="ignore"):
        for p in range(6):
            n, d = np.broadcast_to(P[p, :3], (m, 3)), np.full(m, P[p, 3], f32)
            cloud &= ~np.where(tame, trick_all_behind(n, d, lo, hi), literal_all_behind(n, d, lo, hi))
        strong = tame & (max_corner_s(P, boxes) < pm[None]).any(1)
        alive = np.full(m, 0xFF, np.uint32)
        for k in range(3):
            bits = Cn[:, k].view(np.uint32)
            vals = []
            for u in bits.tolist():
                if u not in vals:
                    vals.append(u)
            masks = [sum(1 << i for i in range(8) if bits[i] == u) for u in vals]
            vv = np.array(vals + [0x7FC00000] * (8 - len(vals)), np.uint32).view(f32)
            mk = np.array(masks + [0] * (8 - len(vals)), np.uint32)
            upto = 8 if len(vals) > 4 else 4
            mask = np.zeros(m, np.uint32)
            for j in range(upto):
                mask |= np.where((vv[j] >= lo[:, k]) & (vv[j] <= hi[:, k]), mk[j], np.uint32(0))
            alive &= mask
    return np.where(cloud, True, np.where(strong, False, alive != 0))


# ---- frusta ------------------------------------------------------------------------------------------------------------------
def oracle_frustum(planes, corners) -> ob.Frustum:
    f = ob.Frustum()
    for p in range(6):
        for k in range(3):
            f.planes[p].n[k] = float(planes[p][k])
        f.planes[p].d = float(planes[p][3])
    for i in range(8):
        for k in range(3):
            f.corners[i][k] = float(corners[i][k])
    return f


class EdgeFrustum:
    """One frustum on both sides: planes / corners as numpy, the oracle's Frustum, the library's fyx_frustum."""

    def __init__(self, name, planes, corners, fo=None, ff=None):
        from fyrox_b200 import frustum_from_numpy

        self.name = name
        self.planes = np.ascontiguousarray(planes, f32).reshape(6, 4)
        self.corners = np.ascontiguousarray(corners, f32).reshape(8, 3)
        self.fo = fo if fo is not None else oracle_frustum(self.planes, self.corners)
        self.ff = ff if ff is not None else frustum_from_numpy(self.planes, self.corners)

    @staticmethod
    def from_vp(name, vp):
        """Built from a view-projection matrix by the oracle and by the library; the two must agree bit for bit."""
        import fyrox_b200 as fb

        fo = ob.frustum_from_vp(vp)
        ff = fb.frustum_from_view_projection_matrix(np.asarray(vp, f32))
        assert fo is not None and ff is not None, name
        P, Cn = ob.frustum_planes_corners(fo)
        Pf, Cf = fb.frustum_to_numpy(ff)
        assert P.tobytes() == Pf.tobytes() and Cn.tobytes() == Cf.tobytes(), f"{name}: host frustum differs from the oracle's"
        return EdgeFrustum(name, P, Cn, fo, ff)

    def intersects(self, boxes):
        return literal_intersects(self.planes, self.corners, boxes)


def _rand_unit(rng):
    v = rng.normal(size=3)
    return v / np.linalg.norm(v)


def perspective_vp(eye, target, up, aspect, fovy, zn, zf):
    view = ob.look_at_rh(tuple(map(float, eye)), tuple(map(float, target)), tuple(map(float, up)))
    return ob.mat4_mul(ob.perspective(float(aspect), float(fovy), float(zn), float(zf)), view)


def edge_frusta(rng):
    """The frustum shapes of the edge tests, eight of them (so that any prefix mixes shapes):
    perspective at random rotations (8 distinct coordinates per axis: the n_ax > 4 half of the fallback runs), two axis-aligned
    cube faces (+-0 normal components, <= 4 distinct coordinates), an orthographic cascade, a far thin frustum (zfar 1e5: pm has a
    large slack), and two filled directly (corners off the planes; one NaN corner) — legal fyx_frustum inputs to fyx_cull."""
    import csm_oracle as co
    from helpers import CUBE_FACES

    out = []
    for r in range(2):
        eye = rng.uniform(-20, 20, 3)
        out.append(EdgeFrustum.from_vp(f"perspective{r}", perspective_vp(eye, eye + _rand_unit(rng), _rand_unit(rng), 16 / 9, np.deg2rad(60.0), 0.1, 150.0)))
    for look, up in (CUBE_FACES[0], CUBE_FACES[3]):
        out.append(EdgeFrustum.from_vp(f"cube{look}", perspective_vp((0, 0, 0), look, up, 1.0, np.pi / 2, 0.01, 120.0)))
    view = co.look_at_lh(np.array([30.0, 40.0, -10.0], f32), np.array([0.0, 0.0, -30.0], f32), np.array([0.0, 1.0, 0.0], f32))
    out.append(EdgeFrustum.from_vp("ortho_cascade", ob.mat4_mul(co.orthographic(-25.0, 25.0, -18.0, 18.0, -40.0, 90.0), view)))
    eye = rng.uniform(-5, 5, 3)
    out.append(EdgeFrustum.from_vp("far_thin", perspective_vp(eye, eye + _rand_unit(rng), _rand_unit(rng), 0.5, np.deg2rad(3.0), 1.0, 1e5)))
    base = EdgeFrustum.from_vp("base", perspective_vp((1, 2, 3), (1.3, 2.1, 2.0), (0, 1, 0), 1.3, np.deg2rad(50.0), 0.5, 60.0))
    off = base.corners + rng.normal(size=(8, 3)).astype(f32) * f32(0.4)  # corners off the planes
    out.append(EdgeFrustum("corners_off_planes", base.planes, off))
    nan_c = base.corners.copy()
    nan_c[6, 1] = np.nan
    out.append(EdgeFrustum("nan_corner", base.planes, nan_c))
    return out


# ---- edge boxes --------------------------------------------------------------------------------------------------------------
def _window(b, k=64):
    """2k+1 consecutive floats centred on b."""
    lo = np.array([b], f32)
    down = [lo[0]]
    up = [lo[0]]
    for _ in range(k):
        down.append(np.nextafter(down[-1], f32(-np.inf)))
        up.append(np.nextafter(up[-1], f32(np.inf)))
    return np.array(down[::-1] + up[1:], f32)


def _sel_hi(n):
    """per axis: does the plane's max corner take the box's maximum (n >= 0, -0 included, as vsel) or its minimum?"""
    return ~(np.asarray(n, f32) < 0)


def _box_from_selected(v, n, ext):
    """Box whose plane-max corner is v: per axis the selected bound is v, the other one ext further along -n (away)."""
    sh = _sel_hi(n)
    lo = np.where(sh, v - ext, v).astype(f32)
    hi = np.where(sh, v, v + ext).astype(f32)
    return np.concatenate([lo, hi])


def _s(P, p, box):
    return max_corner_s(P, box[None])[0, p]


def _plane_boxes(ef, p, rng, tries, point=False):
    """Boxes next to plane p near the middle of its face, outside it, with the max-corner s stepped across 0 one ulp of the
    solved bound at a time.  Returns {label: [boxes]}."""
    P, Cn = ef.planes, ef.corners
    n, d = P[p, :3], P[p, 3]
    k = int(np.argmax(np.abs(n)))
    if not np.isfinite(Cn[list(FACE_CORNERS[p])]).all() or n[k] == 0:
        return {}
    face = Cn[list(FACE_CORNERS[p])].astype(np.float64)
    size = float(np.nanmax(Cn) - np.nanmin(Cn))
    out = {"zero": [], "above": [], "below": []}
    for _ in range(tries):
        q = (rng.dirichlet(np.full(4, 2.0)) @ face).astype(f32)
        ext = np.zeros(3, f32) if point else (size * 10.0 ** rng.uniform(-4, -1.5, 3)).astype(f32)
        v = q.copy()
        # solve n.v + d = 0 for axis k in float64, then scan the floats around it
        rest = sum(float(n[j]) * float(v[j]) for j in range(3) if j != k) + float(d)
        cand = _window(f32(-rest / float(n[k])))
        boxes = []
        for c in cand:
            vv = v.copy()
            vv[k] = c
            boxes.append(_box_from_selected(vv, n, ext))
        boxes = np.array(boxes, f32)
        if not (boxes[:, :3] <= boxes[:, 3:]).all():
            continue
        s = max_corner_s(P, boxes)[:, p]
        z = np.nonzero(s == 0)[0]
        pos = np.nonzero(s > 0)[0]
        neg = np.nonzero(s < 0)[0]
        if z.size:
            out["zero"].append(boxes[z[rng.integers(z.size)]])
        if pos.size:
            out["above"].append(boxes[pos[np.argmin(s[pos])]])
        if neg.size:
            out["below"].append(boxes[neg[np.argmax(s[neg])]])
    return out


def edge_boxes(ef: EdgeFrustum, rng, tries=3):
    """World boxes on the edges of ef's predicate, by class (see the module's docstring).  Every box is (min xyz, max xyz) f32;
    -0 bounds are avoided (a zero translation turns them into +0 in the world box): signed zeros come through the planes and
    corners instead."""
    P, Cn = ef.planes, ef.corners
    pm = dev_frustum_pm(P, Cn)
    size = float(np.nanmax(Cn) - np.nanmin(Cn))
    cls = {c: [] for c in CLASSES}
    for p in range(6):
        b = _plane_boxes(ef, p, rng, tries)
        cls["plane_zero"] += b.get("zero", [])
        cls["plane_above"] += b.get("above", [])
        cls["plane_below"] += b.get("below", [])
        cls["point_plane"] += _plane_boxes(ef, p, rng, 2, point=True).get("zero", [])
        # strong-reject boundary: the max corner is the frustum corner that makes pm, then one bound stepped down until s < pm
        if np.isnan(pm[p]):
            continue
        s_c = max_corner_s(P[p:p + 1].repeat(6, 0), np.concatenate([Cn, Cn], 1))[:, 0]
        j = int(np.nonzero(s_c == pm[p])[0][0])
        n = P[p, :3]
        k = int(np.argmax(np.abs(n)))
        for _ in range(tries):
            ext = (size * 10.0 ** rng.uniform(-4, -1.5, 3)).astype(f32)
            box = _box_from_selected(Cn[j], n, ext)
            assert _s(P, p, box) == pm[p]
            cls["pm_equal"].append(box)
            sel = 3 + k if _sel_hi(n)[k] else k
            other = k if sel == 3 + k else 3 + k
            b2 = box.copy()
            for _ in range(64):
                b2[sel] = np.nextafter(b2[sel], b2[other])
                if _s(P, p, b2) < pm[p]:
                    cls["pm_below"].append(b2.copy())
                    break
    # corner coordinates: the max-corner bounds of each plane through corner i sit on it, or one ulp beyond / short of it
    for i in range(8):
        if not np.isfinite(Cn[i]).all():
            continue
        cls["point_corner"].append(np.concatenate([Cn[i], Cn[i]]))
        for p in range(6):
            if i not in FACE_CORNERS[p]:
                continue
            n = P[p, :3]
            sh = _sel_hi(n)
            ext = (size * 10.0 ** rng.uniform(-4, -1.5, 3)).astype(f32)
            box = _box_from_selected(Cn[i], n, ext)
            cls["corner_on"].append(box)
            for a in range(3):
                sel = 3 + a if sh[a] else a
                away = np.inf if sh[a] else -np.inf  # beyond the corner: it is strictly inside on this axis
                b_in, b_out = box.copy(), box.copy()
                b_in[sel] = np.nextafter(box[sel], f32(away))
                b_out[sel] = np.nextafter(box[sel], f32(-away))
                cls["corner_in"].append(b_in)
                cls["corner_out"].append(b_out)
        # exactly one corner: a small box around it, and one reaching away from the frustum's centre
        centre = np.nanmean(Cn, 0).astype(f32)
        e = (size * 10.0 ** rng.uniform(-5, -3, 3)).astype(f32)
        cls["single_corner"].append(np.concatenate([Cn[i] - e, Cn[i] + e]).astype(f32))
        out_dir = np.sign(Cn[i] - centre).astype(f32)
        far = (Cn[i] + out_dir * f32(size * 0.05)).astype(f32)
        cls["single_corner"].append(np.concatenate([np.minimum(Cn[i], far), np.maximum(Cn[i], far)]).astype(f32))
    fm = np.finfo(f32).max
    c0 = np.nan_to_num(Cn[0], nan=0.0)
    cls["non_tame"] += [np.array(v, f32) for v in (
        [-2e18, c0[1], c0[2], 2e18, c0[1] + 1, c0[2] + 1],
        [c0[0], c0[1], c0[2], c0[0] + 1, 5e18, c0[2] + 1],
        [-np.inf, -np.inf, -np.inf, np.inf, np.inf, np.inf],
        [-np.inf, c0[1], c0[2], c0[0], c0[1] + 1, c0[2] + 1],
        [np.nan, c0[1], c0[2], c0[0] + 1, c0[1] + 1, c0[2] + 1],
        [c0[0], c0[1], c0[2], c0[0] + 1, c0[1] + 1, np.nan],
        [fm, fm, fm, -fm, -fm, -fm],
        [c0[0] + 1, c0[1], c0[2], c0[0], c0[1] + 1, c0[2] + 1],
        [-1e30, -1e30, -1e30, 1e30, 1e30, 1e30],
    )]
    out = {}
    for c, v in cls.items():
        a = np.array(v, f32).reshape(-1, 6)
        # no -0 bound: the world box of an identity child would read +0 there
        a = np.where((a == 0) & np.signbit(a), f32(0.0), a).astype(f32)
        if c in ("corner_in", "corner_out", "single_corner"):
            # next to a corner of a tiny face (a cube face's near plane is 0.02 wide) a box can also reach the neighbouring
            # corners, and a NaN corner holds no coordinate to step from: keep what meets the class's definition
            a = a[classify(P, Cn, a)[c]]
        out[c] = a
    return out


def edge_points(ef: EdgeFrustum, rng, tries=3):
    """Points (zero-extent boxes) on the edges: on each plane (s == 0) and on either side of it, on each frustum corner and one
    ulp off it along every axis, and huge ones (|coordinate| > 1e18).  (m, 3) f32, no -0 coordinate."""
    P, Cn = ef.planes, ef.corners
    pts = []
    for p in range(6):
        for v in _plane_boxes(ef, p, rng, tries, point=True).values():
            pts += [b[:3] for b in v]
    for i in range(8):
        if not np.isfinite(Cn[i]).all():
            continue
        pts.append(Cn[i])
        for a in range(3):
            for way in (-np.inf, np.inf):
                q = Cn[i].copy()
                q[a] = np.nextafter(q[a], f32(way))
                pts.append(q)
    c0 = np.nan_to_num(Cn[0], nan=0.0)
    fm = np.finfo(f32).max  # a light's translation must be finite: huge is as wild as it gets
    pts += [np.array(v, f32) for v in ([2e18, c0[1], c0[2]], [c0[0], -3e19, c0[2]], [fm, c0[1], c0[2]], [-fm, -fm, -fm])]
    a = np.array(pts, f32).reshape(-1, 3)
    return np.where((a == 0) & np.signbit(a), f32(0.0), a).astype(f32)


def interleave(tame, wild, every=8):
    """Non-tame boxes spread lane by lane among tame ones, one in every `every` slots (the non-tame list is cycled), so every
    warp of 32 nodes mixes the max-corner path and the literal path, and the early-exit vote runs over both."""
    out = []
    for i, b in enumerate(tame):
        if i % (every - 1) == 0:
            out.append(wild[(i // (every - 1)) % len(wild)])
        out.append(b)
    return np.array(out, f32).reshape(-1, 6)


def all_boxes(frusta, rng, tries=3, every=8):
    """Edge boxes of every frustum in one shuffled list, non-tame ones interleaved lane by lane."""
    tame, wild = [], []
    for ef in frusta:
        cls = edge_boxes(ef, rng, tries)
        for c, v in cls.items():
            (wild if c == "non_tame" else tame).append(v)
    tame = np.concatenate(tame)
    return interleave(tame[rng.permutation(len(tame))], np.concatenate(wild), every)


def oracle_aabb_intersects(fo, boxes):
    """orc_frustum_is_intersects_aabb over an (m, 6) array."""
    L = ob.lib()
    out = np.empty(len(boxes), bool)
    for i, b in enumerate(np.asarray(boxes, f32).reshape(-1, 6)):
        a = ob.Aabb.make(b[:3], b[3:])
        out[i] = bool(L.orc_frustum_is_intersects_aabb(C.byref(fo), C.byref(a)))
    return out
