"""The float64 skinning reference of skin_cases against the oracle, on the CPU: the oracle's f32 output lies within the
reference's rounding-error bound on every generated edge case, and the bound is tight enough that a kernel with a
slightly wrong weight, a swapped pair of bone indices or a dropped blend shape would fall outside it."""
import numpy as np
import pytest

from skin_cases import LAYOUTS, SkinScene, Surf, oracle_skin, reference_of, skin_f64, within, unpack_vertices, pack_vertices

SPECS = [
    Surf(1, 37, "animated"),
    Surf(3, 129, "packed52", 1),
    Surf(64, 1025, "k16", 7),
    Surf(65, 513, "wide96"),
    Surf(128, 300, "animated", 128),
    Surf(129, 777, "packed52", 0, extreme=True),
    Surf(255, 2000, "wide96", 7, extreme=True),
    Surf(200, 0, "animated"),
    Surf(40, 1500, "k16", 0, extreme=True),
]


@pytest.fixture(scope="module", params=[1, 2])
def scene(request):
    sc = SkinScene(100 + request.param)
    for s in SPECS:
        sc.add(s)
    sc.oracle()
    return sc


def test_generated_cases_reach_the_edges(scene):
    """The generator really produces what the bound and the bit-exact checks are for."""
    seen = {"neg_zero": 0, "subnormal": 0, "overflow": 0, "nan": 0, "non_unit_sum": 0, "one_bone": 0, "last_index": 0}
    for sd in scene.surfaces:
        if not sd.spec.n_verts:
            continue
        pos, nrm, w, bi = unpack_vertices(sd.verts, sd.spec.layout)
        f = np.concatenate([pos, nrm, w], axis=1)
        seen["neg_zero"] += int(((f == 0) & np.signbit(f)).sum())
        seen["subnormal"] += int(((f != 0) & (np.abs(f) < np.finfo(np.float32).tiny)).sum())
        seen["non_unit_sum"] += int((np.abs(w.sum(axis=1) - 1) > 1e-3).sum())
        seen["one_bone"] += int((bi == bi[:, :1]).all(axis=1).sum())
        seen["last_index"] += int((bi == sd.spec.n_bones - 1).any(axis=1).sum())
        p, _ = oracle_skin(scene.oracle_palette(sd), sd)
        seen["overflow"] += int(np.isinf(p).sum())
        seen["nan"] += int(np.isnan(p).sum())
    assert all(v > 0 for v in seen.values()), seen


def test_oracle_lies_within_the_float64_bound(scene):
    checked = 0
    for sd in scene.surfaces:
        pal = scene.oracle_palette(sd)
        pos, nrm = oracle_skin(pal, sd)
        ref = reference_of(pal, sd)
        for name, got, val, bnd in (("positions", pos, ref.pos, ref.pos_bound), ("normals", nrm, ref.nrm, ref.nrm_bound)):
            ok = within(got, val, bnd)
            bad = np.nonzero(~ok.all(axis=1))[0]
            assert bad.size == 0, (f"{sd.spec}: {name} of vertices {bad[:5]} outside the bound: got {got[bad[:3]]}, "
                                   f"want {val[bad[:3]]} +- {bnd[bad[:3]]}")
            checked += int(np.isfinite(bnd).sum())
    assert checked > 0


def test_bound_is_tight_for_ordinary_values():
    """The bound is a handful of ulps of the sum of magnitudes, not a blanket tolerance: with 7 blend shapes the longest
    rounding chain is 8 + 7 + 1 = 16, so on well-scaled data the bound stays within 16.01 u of E."""
    sc = SkinScene(7)
    sd = sc.add(Surf(64, 4000, "animated", 7))
    sc.oracle()
    ref = reference_of(sc.oracle_palette(sd), sd)
    rel = ref.pos_bound / np.maximum(ref.info["Ep"], 1e-30)
    assert np.nanmax(rel[ref.info["Ep"] > 1e-20]) < 16.01 * 2.0 ** -24


def _fraction_outside(pos, nrm, ref, affected):
    ok = within(pos, ref.pos, ref.pos_bound).all(axis=1) & within(nrm, ref.nrm, ref.nrm_bound).all(axis=1)
    return float(1.0 - ok[affected].mean())


@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_bound_catches_a_slightly_wrong_weight(layout):
    sc = SkinScene(11)
    sd = sc.add(Surf(100, 3000, layout))
    sc.oracle()
    pal = sc.oracle_palette(sd)
    ref = reference_of(pal, sd)
    pos, nrm, w, bi = unpack_vertices(sd.verts, layout)
    w2 = w.copy()
    w2[:, 1] = (w2[:, 1].astype(np.float64) * (1 + 2.0 ** -10)).astype(np.float32)
    bad = pack_vertices(np.random.default_rng(0), layout, pos, nrm, w2, bi)
    p2, n2 = oracle_skin(pal, sd, verts=bad)
    affected = (w2[:, 1] != w[:, 1]) & (np.abs(w[:, 1]) > 1e-3) & np.isfinite(ref.pos_bound).all(axis=1)
    assert affected.sum() > 1000
    assert _fraction_outside(p2, n2, ref, affected) > 0.9


def test_bound_catches_swapped_bone_indices():
    sc = SkinScene(12)
    sd = sc.add(Surf(200, 3000, "k16"))
    sc.oracle()
    pal = sc.oracle_palette(sd)
    ref = reference_of(pal, sd)
    pos, nrm, w, bi = unpack_vertices(sd.verts, "k16")
    b2 = bi.copy()
    b2[:, [0, 2]] = bi[:, [2, 0]]
    bad = pack_vertices(np.random.default_rng(0), "k16", pos, nrm, w, b2)
    p2, n2 = oracle_skin(pal, sd, verts=bad)
    affected = (bi[:, 0] != bi[:, 2]) & (np.abs(w[:, 0] - w[:, 2]) > 1e-3) & np.isfinite(ref.pos_bound).all(axis=1)
    assert affected.sum() > 1000
    assert _fraction_outside(p2, n2, ref, affected) > 0.9


def test_bound_catches_a_dropped_blend_shape():
    sc = SkinScene(13)
    sd = sc.add(Surf(64, 3000, "packed52", 7))
    sc.oracle()
    pal = sc.oracle_palette(sd)
    ref = reference_of(pal, sd)
    w100 = sd.w100.copy()
    s = int(np.argmax(w100))  # the shape with the largest weight
    w100[s] = 0.0
    p2, n2 = oracle_skin(pal, sd, weights_w100=w100)
    off = sd.records.view(np.float16)[s, :3000, :6].astype(np.float64)
    pos, nrm, w, bi = unpack_vertices(sd.verts, "packed52")
    affected = (np.abs(off[:, :3]).max(axis=1) > 1e-2) & (np.abs(w).sum(axis=1) > 0.5) & np.isfinite(ref.pos_bound).all(axis=1)
    assert affected.sum() > 500
    assert _fraction_outside(p2, n2, ref, affected) > 0.9


def test_reference_matches_a_direct_matrix_product():
    """skin_f64 against a per-vertex loop over 4x4 matrices (no shared einsum indexing), blend shapes included."""
    sc = SkinScene(14)
    sd = sc.add(Surf(9, 50, "wide96", 3))
    sc.oracle()
    pal = sc.oracle_palette(sd)
    ref = skin_f64(pal, sd.verts, "wide96", (sd.records, sd.w100))
    pos, nrm, w, bi = unpack_vertices(sd.verts, "wide96")
    off = sd.records.view(np.float16).astype(np.float64)
    for v in range(50):
        p = pos[v].astype(np.float64) + sum(off[s, v, 0:3] * float(sd.w100[s]) for s in range(3))
        n = nrm[v].astype(np.float64) + sum(off[s, v, 3:6] * float(sd.w100[s]) for s in range(3))
        want_p, want_n = np.zeros(3), np.zeros(3)
        for k in range(4):
            m = pal[bi[v, k]].astype(np.float64).reshape(4, 4).T  # column-major storage
            want_p += float(w[v, k]) * (m @ np.append(p, 1.0))[:3]
            want_n += float(w[v, k]) * (m[:3, :3] @ n)
        np.testing.assert_allclose(ref.pos[v], want_p, rtol=1e-12, atol=1e-300)
        np.testing.assert_allclose(ref.nrm[v], want_n, rtol=1e-12, atol=1e-300)
