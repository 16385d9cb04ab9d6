"""One pass of push_triangles (renderer/bundle.rs:1177-1243) over its three callers, restated in f32 numpy over the pass's
nodes in the order its DFS visits them: the Dynamic branch of Mesh::collect_render_data (dynamic_batch_oracle), Sprite
(scene/sprite.rs:322-405) and dim2::Rectangle (scene/dim2/rectangle.rs:323-410).

- gates: a quad node pushes nothing in a shadow pass; a sprite nothing without cast_shadows, in any pass;
- a quad node is never an ordinary instance;
- one bundle_map and one last_bundle_id for all three; one shared surface per layout id.
"""
from dataclasses import dataclass

import numpy as np

from dynamic_batch_oracle import _transform, transform_vertices

f32 = np.float32
SPRITE, RECTANGLE = 1, 2
CORNERS = ((0.5, 0.5), (-0.5, 0.5), (-0.5, -0.5), (0.5, -0.5))
STRIDE = {SPRITE: 40, RECTANGLE: 24}
TRIANGLES = np.array([[0, 1, 2], [0, 2, 3]], np.uint32)


@dataclass
class Quad:
    kind: int
    batch_key: int
    layout_id: int
    uv_rect: tuple = (0.0, 0.0, 1.0, 1.0)
    color: tuple = (255, 255, 255, 255)
    size: float = 0.2
    rotation: float = 0.0
    flip_x: bool = False
    flip_y: bool = False

    def record(self):
        """The fyx_sprite record."""
        from fyrox_b200.context import Context

        r = np.zeros(1, Context.SPRITE)
        r[0] = (self.kind, self.batch_key, self.layout_id, int(self.flip_x) | (int(self.flip_y) << 1), self.uv_rect, self.size,
                self.rotation, self.color, 0)
        return r[0]


def quad_vertices(q: Quad, world) -> bytes:
    """The four vertex records (SpriteVertex or RectangleVertex) the node pushes; world: column-major f32[16]."""
    world = np.asarray(world, f32)
    u = [f32(x) for x in q.uv_rect]
    lx, rx, ty, by = u[0], u[0] + u[2], u[1], u[1] + u[3]
    if q.kind == SPRITE:
        tx = [lx if q.flip_x else rx, rx if q.flip_x else lx, rx if q.flip_x else lx, lx if q.flip_x else rx]
    else:
        tx = [rx if q.flip_x else lx, lx if q.flip_x else rx, lx if q.flip_x else rx, rx if q.flip_x else lx]
    tyv = [by if q.flip_y else ty] * 2 + [ty if q.flip_y else by] * 2
    if q.kind == SPRITE:
        pos = np.tile(world[12:15], (4, 1))  # global_position(): no arithmetic
    else:
        pos = _transform(world, np.array([(x, y, 0.0) for x, y in CORNERS], f32), True)
    color = np.array(q.color, np.uint8).tobytes()
    out = b""
    for k, (sx, sy) in enumerate(CORNERS):
        fl = [*pos[k], tx[k], tyv[k]]
        if q.kind == SPRITE:
            fl += [q.size, q.rotation, sx, sy]
        out += np.array(fl, f32).tobytes() + color
    return out


def mixed_pass(nodes, n_surfaces, dynamic, quads, sort_index_of, world_of, shadow=False, cast_shadows=lambda n: True):
    """One pass.  nodes: the pass's nodes (should_be_rendered) in DFS order; dynamic = {(node, ordinal): DynSurface}; quads =
    {node: Quad}; shadow: the pass is a shadow pass; cast_shadows(node).  Returns (batches, pushed) as
    dynamic_batch_oracle.dynamic_pass does."""
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
        q = quads.get(node)
        if q is not None:
            if shadow or (q.kind == SPRITE and not cast_shadows(node)):
                continue
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
