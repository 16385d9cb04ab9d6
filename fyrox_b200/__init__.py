"""fyrox_b200 — H100-native render-prep hot path for Fyrox scenes.

Hierarchical world-transform update, world-AABB recompute, multi-frustum culling with visible-index
compaction, bone-palette build and linear-blend skinning as hand-written sm_90a CUDA kernels behind
a C ABI (include/fyrox_b200.h).  This package is the Python host side: ctypes binding (`Context`),
the mirror of the reference's host interface (`scene`), and the synthetic scene generator.
"""
from . import _lib  # noqa: F401
from ._lib import (  # noqa: F401
    FYX_NONE, LIGHT_DIRECTIONAL, LIGHT_POINT, LIGHT_SPOT, LIGHT_UNKNOWN, NODE_ALIVE, NODE_LIGHT, NODE_STATIC_BATCH, NODE_REFLECTION_PROBE, NODE_CAST_SHADOWS, NODE_DEFAULT, NODE_ENABLED, NODE_FRUSTUM_CULLING, NODE_GLOBAL_ENABLED,
    NODE_GLOBAL_VISIBILITY, NODE_REACHABLE, NODE_RENDERABLE, NODE_VISIBILITY, PASS_SHADOW, UPDATE_ALL, UPDATE_INCREMENTAL,
    PROJECTION_PERSPECTIVE, PROJECTION_ORTHOGRAPHIC, PROJECTION_NONE, PROBE_UPDATE_ONCE, PROBE_UPDATE_EACH_FRAME, OBSERVER_PROBE_FACE, OBSERVER_CAMERA,
)
from .context import (  # noqa: F401
    ANIMATED_VERTEX_LAYOUT, Context, FyxError, PinnedBuffer, frustum_default, frustum_from_numpy,
    frustum_from_view_projection_matrix, frustum_to_numpy, mat4_mul,
)

__all__ = [n for n in dir() if not n.startswith("_")]
