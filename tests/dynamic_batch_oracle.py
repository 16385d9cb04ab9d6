"""Dynamic batching for one pass (RenderDataBundleStorage::push_triangles, renderer/bundle.rs:1177-1243) over its callers: the
Dynamic branch of Mesh::collect_render_data (scene/mesh/mod.rs:804-833) and the quad nodes (sprite_batch_oracle), restated in
numpy over a pass's nodes in the order its DFS visits them.

- bundle_map: (batch key, sort index) -> bundle, in the order of the first push; last_bundle_id, changed only by these
  pushes (one for all callers), decides whether a push extends the last instance (ElementRange::Specific) or starts a new one;
- one shared surface per layout (DynamicSurfaceCache): vertices appended, triangles shifted by the vertex count before them;
- transform_vertex (scene/mesh/mod.rs:109-126) in f32 without fused multiply-add: the position by Matrix4::transform_point
  (orc_mat4_transform_point's arithmetic), the normal and the tangent's xyz by Matrix4::transform_vector (nalgebra:
  transform * v / n with n = row3 . v, no division when n == 0), the tangent's w kept.
"""
from dataclasses import dataclass

import numpy as np

f32 = np.float32
NONE = 0xFFFFFFFF


@dataclass
class DynSurface:
    batch_key: int
    layout_id: int
    layout: tuple  # (stride, position_offset, normal_offset, tangent_offset), NONE = absent
    vertices: bytes
    triangles: np.ndarray  # (n, 3) u32


def _transform(m, v, point):
    """m: column-major f32[16] (affine or not); v: (n, 3) f32.  nalgebra's transform_point / transform_vector."""
    m = np.asarray(m, f32)
    x, y, z = v[:, 0], v[:, 1], v[:, 2]
    n = (m[3] * x + m[7] * y) + m[11] * z
    if point:
        n = n + m[15]
    out = np.empty_like(v)
    for i in range(3):
        t = (m[0 + i] * x + m[4 + i] * y) + m[8 + i] * z
        if point:
            t = t + m[12 + i]
        with np.errstate(all="ignore"):
            out[:, i] = np.where(n != f32(0), t / np.where(n != f32(0), n, f32(1)), t)
    return out


def transform_vertices(raw: bytes, layout, world):
    """The vertex records after transform_vertex; bytes other than the three attributes unchanged."""
    stride, pos, nrm, tan = layout
    rec = np.frombuffer(raw, np.uint8).reshape(-1, stride).copy()
    for off, point in ((pos, True), (nrm, False), (tan, False)):
        if off == NONE or rec.shape[0] == 0:
            continue
        v = np.ascontiguousarray(rec[:, off:off + 12]).view(f32).reshape(-1, 3)
        rec[:, off:off + 12] = _transform(world, v, point).view(np.uint8).reshape(-1, 12)
    return rec.tobytes()


def dynamic_pass(nodes, n_surfaces, dynamic, sort_index_of, world_of, quads=None, shadow=False, cast_shadows=lambda n: True):
    """One pass of push_triangles over its callers: the Dynamic meshes and the quad nodes (sprite_batch_oracle).  nodes: the
    pass's nodes (should_be_rendered) in DFS order; n_surfaces(node) = len(Mesh::surfaces); dynamic = {(node, ordinal):
    DynSurface}; sort_index_of(node), world_of(node) (column-major f32[16]); quads = {node: Quad}, with their gates: shadow (the
    pass is a shadow pass) and cast_shadows(node).  Returns (batches, pushed): batches as Context.dynamic_batches returns them,
    pushed = the (node, ordinal) pairs pushed as ordinary instances; a quad node is never one."""
    bundle_map, bundles, last = {}, [], None
    streams = {}  # layout_id -> [stride, vertex chunks, triangle chunks, vertex count, triangle count]
    pushed = []

    def push(node, batch_key, layout_id, stride, vertices, tri):
        nonlocal last
        si = int(sort_index_of(node))
        key = (batch_key, si)
        if key not in bundle_map:
            bundle_map[key] = len(bundles)
            bundles.append({"batch_key": batch_key, "layout_id": layout_id, "sort_index": si, "instances": []})
        b = bundles[bundle_map[key]]
        st = streams.setdefault(layout_id, [stride, [], [], 0, 0])
        offset = st[4]
        st[1].append(vertices)
        st[2].append(tri + np.uint32(st[3]))
        st[3] += len(vertices) // stride
        st[4] += tri.shape[0]
        if last != key:
            b["instances"].append([node, offset, tri.shape[0]])
            last = key
        else:
            b["instances"][-1][2] += tri.shape[0]

    for node in nodes:
        q = (quads or {}).get(node)
        if q is not None:
            from sprite_batch_oracle import SPRITE, STRIDE, TRIANGLES, quad_vertices

            if not shadow and (q.kind != SPRITE or cast_shadows(node)):
                push(node, q.batch_key, q.layout_id, STRIDE[q.kind], quad_vertices(q, world_of(node)), TRIANGLES)
            continue
        for k in range(n_surfaces(node)):
            d = dynamic.get((node, k))
            if d is None:
                pushed.append((node, k))
                continue
            push(node, d.batch_key, d.layout_id, d.layout[0], transform_vertices(d.vertices, d.layout, world_of(node)),
                 np.asarray(d.triangles, np.uint32).reshape(-1, 3))
    from fyrox_b200.context import Context

    brow, irow = [], []
    for b in bundles:
        brow.append((b["batch_key"], b["layout_id"], len(irow), len(b["instances"]), b["sort_index"]))
        irow.extend((n, o, c, 0) for n, o, c in b["instances"])
    out = {
        "bundles": np.array(brow, Context.DYNAMIC_BUNDLE),
        "instances": np.array(irow, Context.DYNAMIC_INSTANCE),
        "streams": {l: {"stride": st[0], "vertices": np.frombuffer(b"".join(st[1]), np.uint8),
                        "triangles": (np.concatenate(st[2]) if st[2] else np.empty((0, 3), np.uint32)).astype(np.uint32)}
                    for l, st in sorted(streams.items())},
    }
    return out, pushed
