"""The quad nodes among push_triangles' callers (dynamic_batch_oracle.dynamic_pass runs the pass), restated in f32 numpy: Sprite
(scene/sprite.rs:322-405) and dim2::Rectangle (scene/dim2/rectangle.rs:323-410).

- gates: a quad node pushes nothing in a shadow pass; a sprite nothing without cast_shadows, in any pass;
- a quad node is never an ordinary instance;
- one bundle_map and one last_bundle_id with the Dynamic meshes; one shared surface per layout id.
"""
from dataclasses import dataclass

import numpy as np

from dynamic_batch_oracle import _transform

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
