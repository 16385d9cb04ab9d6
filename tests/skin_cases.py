"""Skinning cases shared by the CPU and GPU skinning tests.

* A small scene: the root, a forest of bones with random affine locals (plus a few bones scaled by up to 1e21, a few dead
  nodes) and mesh nodes.
* Surfaces described by (n_bones, n_verts, layout, blend shapes): edge-case vertices packed into one of several vertex
  layouts, their bone lists (with NONE and dead bones) and optional blend shapes.
* The oracle's output for a surface (orc_skin_vertices / orc_skin_vertices_blend on the oracle's palette).
* skin_f64: plain float64 linear-blend skinning of the same inputs with a componentwise bound on the rounding error of
  the f32 computation, so the oracle and the kernel are both checked against arithmetic they do not share.

Importable without a GPU: only `SkinScene.load_into` and `add_to_context`, which the GPU tests call, touch a fyx context.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field

import numpy as np

import fyrox_b200 as fb
import oracle_binding as ob

NONE = 0xFFFFFFFF
FLT_MAX = float(np.finfo(np.float32).max)
U32 = 2.0 ** -24  # unit roundoff of binary32
U64 = 2.0 ** -53  # unit roundoff of binary64
ETA = 2.0 ** -150  # largest absolute error of a product rounded into the subnormal range (half of 2^-149)

# (stride, position, normal, bone weights, bone indices) in bytes; every offset a multiple of 4 (fyx_add_skinned_surface)
LAYOUTS = {
    "animated": (68, 0, 20, 48, 64),  # scene/mesh/vertex.rs AnimatedVertex
    "k16": (76, 0, 28, 56, 72),  # the reference's interleaved test vertex (tests/golden K16)
    "packed52": (52, 40, 24, 8, 0),  # indices first, position last, 4-byte gaps between attributes
    "wide96": (96, 80, 4, 32, 92),  # normal ahead of the weights, position near the end, indices in the last word
}

MAX_BLEND_SHAPES = 128  # FYX_MAX_BLEND_SHAPES
TILE_QUADS = 2048  # four-vertex groups per skinning tile (commit_surfaces)


@dataclass
class Surf:
    """One surface: palette size, vertex count, vertex layout, number of blend shapes, and whether some vertices and
    bones are scaled so far that products overflow f32."""
    n_bones: int
    n_verts: int
    layout: str = "animated"
    n_shapes: int = 0
    extreme: bool = False


@dataclass
class SurfaceData:
    spec: Surf
    mesh: int
    bones: np.ndarray  # uint32 bone nodes (NONE allowed)
    verts: np.ndarray  # uint8 (n_verts, stride)
    records: np.ndarray | None = None  # uint16 (n_shapes, layer_stride, 9): binary16 position / normal / tangent offsets
    weights: np.ndarray | None = None  # f32 BlendShape::weight (0..100)
    oracle_surface: int = -1  # index of the surface on its mesh node in the oracle graph

    @property
    def w100(self):
        """The per-shape factors the shader uses: weight / 100 rounded to f32 (scene/mesh/mod.rs:794-798)."""
        return (self.weights.astype(np.float32) / np.float32(100.0)).astype(np.float32)


def vertex_layout(name) -> ob.VertexLayout:
    return ob.VertexLayout(*LAYOUTS[name])


def gamma(n, u=U32):
    """gamma_n = n u / (1 - n u): the relative error bound of a chain of n roundings (Higham, Lemma 3.1)."""
    return n * u / (1.0 - n * u)


# ---- vertices ----------------------------------------------------------------------------------------------
def pack_vertices(rng, layout, pos, nrm, w, bi):
    stride, po, no, wo, io = LAYOUTS[layout]
    nv = pos.shape[0]
    rec = rng.integers(0, 256, (nv, stride), dtype=np.uint8)  # bytes no attribute covers are noise
    rec[:, po:po + 12] = np.ascontiguousarray(pos, np.float32).view(np.uint8).reshape(nv, 12)
    rec[:, no:no + 12] = np.ascontiguousarray(nrm, np.float32).view(np.uint8).reshape(nv, 12)
    rec[:, wo:wo + 16] = np.ascontiguousarray(w, np.float32).view(np.uint8).reshape(nv, 16)
    rec[:, io:io + 4] = np.ascontiguousarray(bi, np.uint8)
    return rec


def unpack_vertices(verts, layout):
    stride, po, no, wo, io = LAYOUTS[layout]
    rec = np.ascontiguousarray(verts, np.uint8).reshape(-1, stride)

    def f32(o, k):
        return np.ascontiguousarray(rec[:, o:o + 4 * k]).view(np.float32).reshape(-1, k)

    return f32(po, 3), f32(no, 3), f32(wo, 4), np.ascontiguousarray(rec[:, io:io + 4])


def make_vertices(rng, n_verts, n_bones, special=(), extreme=False):
    """Positions / normals / weights / u8 indices with the edges of linear-blend skinning mixed in:
    zero weights and weights that do not sum to 1 (some negative), all four influences on one bone, indices 0 and
    n_bones - 1 in every lane, the palette entries in `special` (NONE / dead bones), -0.0 and f32 subnormals in
    positions, normals and weights; with `extreme`, positions up to ~1e18."""
    nv = n_verts
    pos = rng.uniform(-3, 3, (nv, 3)).astype(np.float32)
    nrm = rng.normal(size=(nv, 3)).astype(np.float32)
    w = rng.random((nv, 4)).astype(np.float32)
    w /= w.sum(axis=1, keepdims=True)
    bi = rng.integers(0, n_bones, (nv, 4)).astype(np.uint8)
    if nv == 0:
        return pos, nrm, w, bi
    v = np.arange(nv)
    r = rng.random(nv)
    # weights
    w[r < 0.05, 2:] = 0.0
    w[(r >= 0.05) & (r < 0.08)] = 0.0  # no influence at all
    scale = np.where((r >= 0.08) & (r < 0.2), rng.uniform(0.2, 3.0, nv), 1.0).astype(np.float32)
    w *= scale[:, None]  # sums other than 1
    neg = (r >= 0.2) & (r < 0.23)
    w[neg, 3] = -w[neg, 3]
    # indices: all four on one bone; 0 and n_bones - 1 in lane (v mod 11) for v mod 11 < 8
    same = (r >= 0.3) & (r < 0.36)
    bi[same] = bi[same, :1]
    m11 = v % 11
    for lane in range(4):
        bi[m11 == lane, lane] = 0
        bi[m11 == 4 + lane, lane] = n_bones - 1
    for k, e in enumerate(special):  # NONE / dead palette entries (identity) in a lane each
        sel = (v % 13) == 9 + k % 4
        bi[sel, k % 4] = e
    # signed zeros and subnormals
    q = rng.random((nv, 10))
    tiny = np.float32(1e-40) * rng.uniform(-1, 1, (nv, 10)).astype(np.float32)  # binary32 subnormals
    f = np.concatenate([pos, nrm, w], axis=1)
    f[q < 0.02] = -0.0
    sub = (q >= 0.02) & (q < 0.04)
    f[sub] = tiny[sub]
    f[(q >= 0.04) & (q < 0.045)] = np.float32(1.4e-45)  # the smallest subnormal
    pos, nrm, w = f[:, 0:3].copy(), f[:, 3:6].copy(), f[:, 6:10].copy()
    if extreme:
        big = rng.random(nv) < 0.25
        pos[big] *= (10.0 ** rng.uniform(0, 18, (int(big.sum()), 1))).astype(np.float32)
    return pos.astype(np.float32), nrm.astype(np.float32), w.astype(np.float32), bi


def make_blend_shapes(rng, n_verts, n_shapes):
    """BlendShapesContainer records (n_shapes, layer_stride >= n_verts, 9 binary16) and weights in 0..100."""
    stride = n_verts + int(rng.integers(0, 6))
    off = (rng.normal(size=(n_shapes, stride, 9)) * 0.2).astype(np.float16)
    off[rng.random(off.shape) < 0.4] = 0
    if n_verts:
        off[0, 0, :3] = [np.float16(6.1e-5), np.float16(-0.0), np.float16(5.96e-8)]  # smallest normal, -0, a subnormal
    w = rng.uniform(0, 100, n_shapes).astype(np.float32)
    if n_shapes > 1:
        w[-1] = 0.0
        w[0] = 100.0
    return off.view(np.uint16), w


# ---- scene -------------------------------------------------------------------------------------------------
def _affine(rng, scale_range=(0.5, 1.5), t_range=20.0):
    t = ob.Transform()
    ob.lib().orc_transform_identity(t)
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    t.local_position[:] = rng.uniform(-t_range, t_range, 3).astype(np.float32).tolist()
    t.local_rotation[:] = q.astype(np.float32).tolist()
    t.local_scale[:] = rng.uniform(*scale_range, 3).astype(np.float32).tolist()
    m = np.empty(16, np.float32)
    ob.lib().orc_transform_calculate_local(t, ob.fp(m))
    return m


class SkinScene:
    """Root (node 0), `n_bones` bones in a random forest under it, 4 huge bones (scale 1e19..1e21, children of the
    root), 3 dead nodes, then `n_meshes` mesh nodes.  Inverse bind poses are per node, as in the reference.  The oracle
    graph holds each surface's bone list only (for orc_mesh_bone_matrices); oracle_skin skins the vertices on that
    palette, with the blend shapes when the surface has any."""

    def __init__(self, seed, n_bones=300, n_meshes=48):
        rng = self.rng = np.random.default_rng(seed)
        self.bone_nodes = np.arange(1, 1 + n_bones, dtype=np.uint32)
        self.huge_nodes = np.arange(1 + n_bones, 5 + n_bones, dtype=np.uint32)
        self.dead_nodes = np.arange(5 + n_bones, 8 + n_bones, dtype=np.uint32)
        self.mesh_nodes = np.arange(8 + n_bones, 8 + n_bones + n_meshes, dtype=np.uint32)
        n = self.n = 8 + n_bones + n_meshes
        parent = np.zeros(n, np.uint32)
        parent[0] = NONE
        for i, b in enumerate(self.bone_nodes):  # a parent among the earlier bones or the root: depth ~ log n
            parent[b] = 0 if i == 0 or rng.random() < 0.15 else self.bone_nodes[rng.integers(max(0, i - 40), i)]
        flags = np.full(n, fb.NODE_DEFAULT, np.uint32)
        flags[self.dead_nodes] = 0
        flags[self.mesh_nodes] |= fb.NODE_RENDERABLE
        local = np.tile(np.eye(4, dtype=np.float32).reshape(16), (n, 1))
        for b in self.bone_nodes:
            local[b] = _affine(rng)
        for k, b in enumerate(self.huge_nodes):
            local[b] = _affine(rng, (10.0 ** (19 + k * 0.7), 10.0 ** (19 + k * 0.7) * 1.5), 1e4)
        for m in self.mesh_nodes:
            local[m] = _affine(rng)
        self.parent, self.flags, self.local = parent, flags, local
        self.inv_bind = np.tile(np.eye(4, dtype=np.float32).reshape(16), (n, 1))
        for b in np.concatenate([self.bone_nodes, self.huge_nodes, self.dead_nodes]):
            self.inv_bind[b] = _affine(rng, t_range=5.0)
        self.aabb = np.tile(np.array([-0.5, -0.5, -0.5, 0.5, 0.5, 0.5], np.float32), (n, 1))
        self.surfaces: list[SurfaceData] = []
        self.og = None

    # -- surfaces --
    def make_surface(self, spec: Surf, mesh=None) -> SurfaceData:
        rng = self.rng
        nb = spec.n_bones
        bones = rng.choice(self.bone_nodes, nb, replace=False).astype(np.uint32)
        special = []
        if nb >= 4:  # one NONE and one dead palette entry
            j = rng.choice(nb, 2, replace=False)
            bones[j[0]] = NONE
            bones[j[1]] = self.dead_nodes[rng.integers(len(self.dead_nodes))]
            special = [int(j[0]), int(j[1])]
        if spec.extreme and nb >= 8:
            j = rng.choice(np.setdiff1d(np.arange(nb), special), 4, replace=False)
            bones[j] = self.huge_nodes
            special += [int(x) for x in j]
        pos, nrm, w, bi = make_vertices(rng, spec.n_verts, nb, special, spec.extreme)
        verts = pack_vertices(rng, spec.layout, pos, nrm, w, bi)
        records = weights = None
        if spec.n_shapes:
            records, weights = make_blend_shapes(rng, spec.n_verts, spec.n_shapes)
        if mesh is None:
            mesh = int(self.mesh_nodes[len(self.surfaces) % len(self.mesh_nodes)])
        return SurfaceData(spec, mesh, bones, verts, records, weights)

    def add(self, spec: Surf) -> SurfaceData:
        """A new surface, registered in the oracle graph when it exists (for its palette)."""
        sd = self.make_surface(spec)
        self.surfaces.append(sd)
        if self.og is not None:
            sd.oracle_surface = self.og.add_surface(sd.mesh, sd.bones)
        return sd

    # -- oracle side --
    def oracle(self) -> ob.Graph:
        og = ob.Graph.build(self.parent, self.flags, None, self.local, self.aabb)
        for b in np.concatenate([self.bone_nodes, self.huge_nodes]):
            og.set_inv_bind(int(b), self.inv_bind[b])
        for sd in self.surfaces:
            sd.oracle_surface = og.add_surface(sd.mesh, sd.bones)
        og.L.orc_graph_drop_messages(og.h)
        og.update_hierarchical_data()
        self.og = og
        return og

    def oracle_palette(self, sd: SurfaceData):
        return self.og.bone_matrices(sd.mesh, sd.oracle_surface, sd.spec.n_bones)

    def move_bones(self, count):
        """New random locals for `count` ordinary bones; applied to the oracle graph.  Returns (idx, m16) for the context."""
        idx = np.sort(self.rng.choice(self.bone_nodes, count, replace=False)).astype(np.uint32)
        m = np.stack([_affine(self.rng) for _ in idx]).astype(np.float32)
        self.local[idx] = m
        if self.og is not None:
            for i, mm in zip(idx, m):
                self.og.set_local_matrix(int(i), mm)
            self.og.update_hierarchical_data()
        return idx, m

    def new_weights(self, sd: SurfaceData):
        w = self.rng.uniform(0, 100, sd.spec.n_shapes).astype(np.float32)
        w[self.rng.random(w.size) < 0.2] = 0.0
        sd.weights = w
        return w

    # -- context side (GPU tests) --
    def load_into(self, ctx):
        ctx.set_topology(self.parent, self.flags, None, self.aabb, root=0)
        ctx.set_local_matrices(self.local)
        return [add_to_context(ctx, self, sd) for sd in self.surfaces]


def add_to_context(ctx, scene: SkinScene, sd: SurfaceData):
    ib = scene.inv_bind[np.where(sd.bones == NONE, 0, sd.bones)]
    verts = sd.verts.reshape(-1) if sd.spec.n_verts else None
    layout = fb._lib.fyx_vertex_layout(*LAYOUTS[sd.spec.layout])
    sid = ctx.add_skinned_surface(sd.mesh, sd.bones, ib, verts, layout=layout)
    if sd.spec.n_shapes:
        ctx.set_blend_shapes(sid, sd.records, sd.weights)
    return sid


def oracle_skin(pal, sd: SurfaceData, weights_w100=None, verts=None):
    """The oracle's skinned positions and normals of a surface for palette `pal` (blend shapes first when it has any)."""
    nv = sd.spec.n_verts
    pos = np.empty((nv, 3), np.float32)
    nrm = np.empty((nv, 3), np.float32)
    if not nv:
        return pos, nrm
    L = ob.lib()
    lay = vertex_layout(sd.spec.layout)
    v = np.ascontiguousarray(sd.verts if verts is None else verts)
    p = np.ascontiguousarray(pal, np.float32).reshape(-1)
    if sd.spec.n_shapes:
        rec = np.ascontiguousarray(sd.records)
        w = np.ascontiguousarray(sd.w100 if weights_w100 is None else weights_w100, np.float32)
        L.orc_skin_vertices_blend(ob.fp(p), nv, v.ctypes.data_as(C.c_void_p), C.byref(lay), rec.shape[0], rec.ctypes.data_as(C.c_void_p),
                                  rec.shape[1], ob.fp(w), ob.fp(pos.reshape(-1)), ob.fp(nrm.reshape(-1)))
    else:
        L.orc_skin_vertices(ob.fp(p), nv, v.ctypes.data_as(C.c_void_p), C.byref(lay), ob.fp(pos.reshape(-1)), ob.fp(nrm.reshape(-1)))
    return pos, nrm


def tile_starts(specs):
    """First four-vertex group of every skinning tile when the surfaces are added in this order (commit_surfaces:
    each surface starts at a multiple of 4 vertices, a surface of q groups makes ceil(q / 2048) tiles of
    ceil(q / tiles) groups).  Returns (absolute group, group within the surface) per tile."""
    out, off = [], 0
    for s in specs:
        q = (s.n_verts + 3) // 4
        if q:
            nt = (q + TILE_QUADS - 1) // TILE_QUADS
            per = (q + nt - 1) // nt
            out += [(off + t * per, t * per) for t in range(nt)]
        off += q
    return out


# ---- float64 reference ---------------------------------------------------------------------------------------
@dataclass
class SkinRef:
    pos: np.ndarray  # (n, 3) float64
    nrm: np.ndarray
    pos_bound: np.ndarray  # (n, 3) float64 error bound; NaN where an f32 intermediate may overflow (checked bit-exactly only)
    nrm_bound: np.ndarray
    info: dict = field(default_factory=dict)


def skin_f64(palette, verts, layout, shapes=None) -> SkinRef:
    """Linear-blend skinning in float64 of f32 inputs: positions sum_k w_k (M_k p), normals sum_k w_k (mat3(M_k) n), with
    blend shapes p += o_s w_s (w_s = weight / 100 as the f32 the shader gets) added first.

    Error bound of the f32 evaluation (the oracle's and the kernel's operation order, one rounding per * and +):
      t_i = ((m_i0 x + m_i1 y) + m_i2 z) + m_i3   the term m_i0 x passes 1 product + 3 sums      = 4 roundings
      acc_i += t_i * w_k, acc starting at 0       1 product, then at most 3 sums (0 + a is exact) = 4 more
    so every exact product in the sum passes at most n = 8 roundings and |fl - exact| <= gamma_8 * E with
      E = sum_k |w_k| (|m_i0 x| + |m_i1 y| + |m_i2 z| + |m_i3|)        (Higham, Accuracy and Stability, 3.1-3.5).
    Normals lack the m_i3 sum: n = 7.  S blend shapes make p_j + sum_s o_s w_s with at most S + 1 roundings per term:
    |p^ - P| <= gamma_{S+1} A with A = |p| + sum_s |o_s w_s|; skinning p^ instead of P gives
    (1 + gamma_n)(1 + gamma_{S+1}) - 1 <= gamma_{n+S+1} relative to E evaluated with A in place of |p|.
    Gradual underflow (the library is built -ftz=false): a sum that lands in the subnormal range is exact; a product
    may err by ETA = 2^-150 absolute.  The 3 coordinate products of bone k reach the result times |w_k|, the weight
    product directly, a blend product times sum_k |w_k| |m_ij|; all of it times (1 + gamma_n) for later roundings.
    The float64 evaluation adds gamma_{n+S+4}(u = 2^-53) E (f32 x f32 products are exact in f64).
    Components where E, an unweighted bone term or the blended input reach FLT_MAX / 2 may overflow an f32
    intermediate (then inf * 0 = NaN is possible): their bound is NaN and they are compared bit-for-bit only."""
    pos, nrm, w, bi = unpack_vertices(verts, layout)
    nv = pos.shape[0]
    P = pos.astype(np.float64)
    N = nrm.astype(np.float64)
    AP, AN = np.abs(P), np.abs(N)
    S = 0
    if shapes is not None:
        rec, w100 = shapes
        S = int(rec.shape[0])
        off = np.ascontiguousarray(rec).view(np.float16)[:, :nv, :6].astype(np.float64)
        for s in range(S):
            ws = float(np.float32(w100[s]))
            P = P + off[s, :, 0:3] * ws
            N = N + off[s, :, 3:6] * ws
            AP = AP + np.abs(off[s, :, 0:3] * ws)
            AN = AN + np.abs(off[s, :, 3:6] * ws)
    M = np.asarray(palette, np.float32).reshape(-1, 4, 4).astype(np.float64).transpose(0, 2, 1)  # M[b, row, col]
    idx = bi.astype(np.int64)
    Lin = M[idx][:, :, :3, :3]  # (nv, 4, 3, 3)
    T = M[idx][:, :, :3, 3]  # (nv, 4, 3)
    W = w.astype(np.float64)
    aW = np.abs(W)
    tp = np.einsum("vkij,vj->vki", Lin, P) + T
    tn = np.einsum("vkij,vj->vki", Lin, N)
    ref_p = np.einsum("vk,vki->vi", W, tp)
    ref_n = np.einsum("vk,vki->vi", W, tn)
    aL = np.abs(Lin)
    bone_p = np.einsum("vkij,vj->vki", aL, AP) + np.abs(T)  # unweighted per-bone magnitudes
    bone_n = np.einsum("vkij,vj->vki", aL, AN)
    Ep = np.einsum("vk,vki->vi", aW, bone_p)
    En = np.einsum("vk,vki->vi", aW, bone_n)
    lin_w = np.einsum("vk,vkij->vij", aW, aL).sum(axis=2)  # sum_k |w_k| sum_j |m_ij|
    under = (3.0 * aW + 1.0).sum(axis=1)[:, None] + S * lin_w

    def bound(E, B, A, n):
        nn = n + (S + 1 if S else 0)
        b = gamma(nn) * E + (1.0 + gamma(nn)) * ETA * under + gamma(nn + 4, U64) * E
        ok = (E < FLT_MAX / 2) & (B.max(axis=1) < FLT_MAX / 2) & (A.max(axis=1, keepdims=True) < FLT_MAX / 2)
        return np.where(ok, b, np.nan)

    return SkinRef(ref_p, ref_n, bound(Ep, bone_p, AP, 8), bound(En, bone_n, AN, 7), {"Ep": Ep, "En": En, "n_shapes": S})


def within(got, value, bnd):
    """Componentwise: |got - value| <= bound, or the component is only checked bit-exactly (NaN bound)."""
    g = np.asarray(got, np.float32).astype(np.float64)
    with np.errstate(invalid="ignore"):
        return np.isnan(bnd) | (np.abs(g - value) <= bnd)


def reference_of(pal, sd: SurfaceData) -> SkinRef:
    shapes = (sd.records, sd.w100) if sd.spec.n_shapes else None
    return skin_f64(pal, sd.verts, sd.spec.layout, shapes)
