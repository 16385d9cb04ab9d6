/*
 * fyrox_b200.h — C ABI of libfyrox_b200: Fyrox's per-frame render-prep hot path on H100 (sm_90a).
 *
 * The reference (Rust) has no FFI seam on this path (SURVEY.md §0 D6, §8b); these entry points are what
 * a Rust `-sys` shim would bind.  Each one names the reference interface it replaces (paths relative
 * to the Fyrox tree).  See INTEGRATION.md for the Rust-side binding and call sites.
 *
 * Conventions
 *  - extern "C", plain pointers and sizes; no exceptions cross the boundary.
 *  - Return value: FYX_OK (0) or a negative fyx_status; fyx_last_error(ctx) gives a message.  This mirrors
 *    the reference's "log and continue" policy: invalid handles are skipped, never fatal
 *    (scene/graph/mod.rs:1167,1206; scene/mesh/mod.rs:785-791).
 *  - Node index i == Handle::index() of the node in Graph's Pool<Node>; capacity == Pool::get_capacity()
 *    (fyrox-core/src/pool/mod.rs:1104).  0xFFFFFFFF == Handle::NONE.
 *  - Matrices are 16 f32, column-major — nalgebra's Matrix4<f32> memory layout (bytemuck-castable).
 *    Only affine matrices (bottom row exactly 0,0,0,1) are accepted: that is all Transform::matrix()
 *    can produce (scene/transform.rs:476-539).
 *  - Caller owns every pointer it passes in; inputs are consumed before the call returns.  Pointers
 *    returned by fyx_get_visible* are library-owned and valid until the next fyx_cull*, fyx_render_prep or
 *    fyx_destroy on that context.
 *  - One fyx_ctx is used from one thread at a time (the engine's game-loop thread, engine/executor.rs:470-517).
 *  - There is no CPU fallback: every compute entry point runs hand-written sm_90a kernels and fails
 *    with FYX_ERR_CUDA if no device is usable.
 */
#ifndef FYROX_B200_H
#define FYROX_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FYX_ABI_VERSION 2u
#define FYX_NONE 0xFFFFFFFFu
#define FYX_MAX_FRUSTA 8u      /* frusta per fyx_cull call: 1 camera, 3 CSM cascades, 6 cube faces (SURVEY §0 D5) */
#define FYX_MAX_BONES 255u     /* fyrox-material/src/shader/mod.rs:613; u8 indices scene/mesh/vertex.rs:154 */

typedef enum fyx_status {
    FYX_OK = 0,
    FYX_ERR_INVALID_ARGUMENT = -1,
    FYX_ERR_CUDA = -2,            /* CUDA runtime/driver error, or no sm_90 device */
    FYX_ERR_OUT_OF_MEMORY = -3,
    FYX_ERR_NOT_AFFINE = -4,      /* a matrix with a bottom row other than (0,0,0,1) or a non-finite entry */
    FYX_ERR_TOPOLOGY = -5,        /* cycle in parent[] / parent out of range */
    FYX_ERR_STATE = -6,           /* call order (e.g. cull before set_topology) */
    FYX_ERR_NCCL = -7,
    FYX_ERR_UNSUPPORTED = -8
} fyx_status;

/* Per-node flag word (inputs).  Bits 0..3 are Base's fields (scene/base.rs:412-432 and TrackedProperty
 * visibility/enabled :441-450), bit 4 the pool record's liveness, bit 5 "this node kind emits render
 * data and is frustum-tested" (Mesh::collect_render_data, scene/mesh/mod.rs:691-698). */
#define FYX_NODE_VISIBILITY      (1u << 0)
#define FYX_NODE_ENABLED         (1u << 1)
#define FYX_NODE_FRUSTUM_CULLING (1u << 2)
#define FYX_NODE_CAST_SHADOWS    (1u << 3)
#define FYX_NODE_ALIVE           (1u << 4)
#define FYX_NODE_RENDERABLE      (1u << 5)
#define FYX_NODE_LIGHT           (1u << 6)  /* the node is a BaseLight (point / spot / directional): fyx_cull_lights */
#define FYX_NODE_STATIC_BATCH    (1u << 7)  /* Mesh with BatchingMode::Static: when it is rendered for a frustum its children are
                                            * not visited for that frustum (RdcControlFlow::Break, scene/mesh/mod.rs:701-725) and its
                                            * instance carries the identity world matrix */
#define FYX_NODE_REFLECTION_PROBE (1u << 15) /* the node is a ReflectionProbe: fyx_select_reflection_probes */
#define FYX_NODE_INPUT_MASK      0x80FFu
/* Computed bits, readable through fyx_get_global_flags (Base::global_visibility / is_globally_enabled,
 * scene/base.rs:751-770) */
#define FYX_NODE_GLOBAL_VISIBILITY (1u << 8)
#define FYX_NODE_GLOBAL_ENABLED    (1u << 9)
#define FYX_NODE_REACHABLE         (1u << 10)  /* reached by the DFS from Graph::root (renderer/bundle.rs:1004) */

/* fyx_update_transforms flags */
#define FYX_UPDATE_INCREMENTAL 0u  /* Graph::update semantics: only sub-trees under changed nodes (process_node_messages) */
#define FYX_UPDATE_ALL         1u  /* Graph::update_hierarchical_data semantics: everything from the root */

/* fyx_cull pass flags */
#define FYX_PASS_SHADOW (1u << 0)  /* renderer::is_shadow_pass ⇒ nodes without cast_shadows are dropped */

typedef struct fyx_ctx fyx_ctx;

typedef struct fyx_config {
    uint32_t struct_size;   /* = sizeof(fyx_config) */
    int32_t  device;        /* CUDA device ordinal; -1 = current device */
    void    *stream;        /* cudaStream_t to launch on; NULL = the context creates its own */
    uint32_t flags;         /* reserved, 0 */
} fyx_config;

/* Frustum as fyrox-math/src/frustum.rs:26-30: planes 0 left,1 right,2 top,3 bottom,4 far,5 near, each
 * (nx,ny,nz,d) normalised; 8 corners in the order of frustum.rs:70-79. */
typedef struct fyx_frustum {
    float planes[6][4];
    float corners[8][3];
} fyx_frustum;

/* Where the attributes live inside one interleaved vertex (VertexBuffer layout, scene/mesh/buffer.rs:404-414).
 * AnimatedVertex (scene/mesh/vertex.rs:140-210): stride 68, position 0, normal 20, weights 48, indices 64. */
typedef struct fyx_vertex_layout {
    uint32_t stride;
    uint32_t position_offset;      /* f32 x3 */
    uint32_t normal_offset;        /* f32 x3 */
    uint32_t bone_weights_offset;  /* f32 x4 */
    uint32_t bone_indices_offset;  /* u8  x4 */
} fyx_vertex_layout;

/* Device-side durations of the stages run by the last fyx_render_prep / individual calls, in ms
 * (the GPU path's counterpart of GraphPerformanceStatistics, scene/graph/mod.rs:94-122).
 * Per-stage values are recorded by SYNCHRONOUS frames only: the events sit between the kernels of the frame's
 * programmatic-dependent-launch chain and would serialise it, so FYX_FRAME_ASYNC frames fill total_ms alone. */
typedef struct fyx_timings {
    float upload_ms;    /* H2D + scatter of changed local matrices / flags */
    float update_ms;    /* hierarchy + world AABB (+ fused cull) */
    float cull_ms;      /* stand-alone cull */
    float palette_ms;
    float skin_ms;
    float readback_ms;  /* D2H of visible counts + lists */
    float total_ms;
} fyx_timings;

/* ---- life cycle -------------------------------------------------------------------------- */
uint32_t    fyx_abi_version(void);
int32_t     fyx_create(const fyx_config *cfg, fyx_ctx **out_ctx);
void        fyx_destroy(fyx_ctx *ctx);
const char *fyx_last_error(const fyx_ctx *ctx);   /* ctx may be NULL: last error of fyx_create on this thread */
int32_t     fyx_sync(fyx_ctx *ctx);
/* Pinned host memory for zero-staging transfers (optional; any host pointer is accepted everywhere). */
void       *fyx_host_alloc(size_t bytes);
void        fyx_host_free(void *p);

/* ---- host-side math on the path (tiny, per frustum) ---------------------------------------- */
/* Frustum::from_view_projection_matrix (fyrox-math/src/frustum.rs:54-82) with Plane::from_abcd /
 * intersection_point (plane.rs:63-75,94-102).  Returns FYX_ERR_INVALID_ARGUMENT where the reference
 * returns None (a zero-length plane normal); callers then use fyx_frustum_default like
 * renderer/bundle.rs:893-896 (`unwrap_or_default`). */
int32_t fyx_frustum_from_view_projection_matrix(const float vp_m16[16], fyx_frustum *out);
void    fyx_frustum_default(fyx_frustum *out);                      /* frustum.rs:32-43 */
/* Matrix4 * Matrix4 in nalgebra's accumulation order (projection * view, renderer/bundle.rs:894). */
void    fyx_mat4_mul(const float a_m16[16], const float b_m16[16], float out_m16[16]);

/* ---- scene description (on load / when the hierarchy changes) ------------------------------ */
/* Replaces the pointer graph walked by Graph::update_hierarchical_data (scene/graph/mod.rs:1272-1292):
 * parent[i] = Base::parent index or FYX_NONE; flags[i] = FYX_NODE_* input bits; render_mask[i] =
 * Base::render_mask (NULL = all ones); local_aabb_minmax = 6 f32 per node (min xyz, max xyz) —
 * NodeTrait::local_bounding_box (Mesh: scene/mesh/mod.rs:631-656; others the unit box, scene/base.rs:733-735;
 * NULL = unit box everywhere).  root = Graph::root index.  global_index (optional, NULL = identity) is the
 * value written to visible lists for node i — used when a context holds one shard of a larger graph.
 * Marks every node changed (like Base::on_connected_to_graph, scene/base.rs:520-540): the next update recomputes
 * every global matrix and world box.
 * What the call keeps: everything that is per node but not an argument here — local matrices, TRS records, transform
 * statics, bundle ids, LOD ranges, light sources, CSM options, cameras, reflection probes, node surfaces, skinned surfaces
 * and animations — stays with its node index (the data moves to the node's new place on the device); a node index that was
 * not alive before the call starts from the defaults (identity local matrix ...).  The DFS order is kept while `capacity` is unchanged.  So the add / link / remove sequence of
 * INTEGRATION.md is: fyx_set_topology with the new columns, then upload the matrices of the NEW or changed nodes only. */
int32_t fyx_set_topology(fyx_ctx *ctx, uint32_t capacity, uint32_t root, const uint32_t *parent,
                         const uint32_t *flags, const uint32_t *render_mask, const float *local_aabb_minmax,
                         const uint32_t *global_index);

/* Optional.  preorder_rank[i] = position of node i in the pre-order DFS from the root in `children` order — the
 * order Graph::update_global_transform_recursively visits nodes (scene/graph/mod.rs:1199-1241).  Only one thing
 * depends on it: Mesh::on_global_transform_changed (scene/mesh/mod.rs:676-682) folds each bone's position AS STORED
 * when the mesh is visited, so a bone that comes later in that order contributes its position from before the
 * update.  With the order given, such bones are snapshotted before every update and the skinned-mesh boxes equal
 * the reference's; without it (or NULL) every bone contributes its new position — identical whenever skeletons
 * precede their meshes.  Kept by fyx_set_topology while the capacity is unchanged. */
int32_t fyx_set_dfs_order(fyx_ctx *ctx, uint32_t capacity, const uint32_t *preorder_rank);

/* Transform::matrix() of `count` nodes (scene/transform.rs:544-550); idx NULL = nodes 0..count-1.
 * Equivalent of `local_transform_mut()` → NodeMessageKind::TransformChanged (scene/base.rs:343-352). */
int32_t fyx_set_local_matrices(fyx_ctx *ctx, uint32_t count, const uint32_t *idx, const float *m16_colmajor);
/* The same, but the library evaluates Transform::calculate_local_transform (scene/transform.rs:421-540) on the
 * device from the Transform's fields instead of receiving the 64-byte matrix: 40 B per changed node go over
 * PCIe instead of 64.  position / rotation (unit quaternion i,j,k,w) / scale are what animation writes every
 * frame (AnimationPose::apply, scene/animation/mod.rs:147-179); the remaining fields of Transform rarely
 * change and are set once with fyx_set_transform_statics (default: identity pre-rotation and post-rotation
 * matrix, zero pivots/offsets — TransformBuilder's defaults, scene/transform.rs:176-200). */
typedef struct fyx_trs {
    float position[3];
    float rotation[4];
    float scale[3];
} fyx_trs;
typedef struct fyx_transform_statics {
    float pre_rotation[4];            /* unit quaternion i,j,k,w */
    float post_rotation_matrix[9];    /* column-major 3x3: Transform::post_rotation_matrix (inverse of the post rotation, :160-172) */
    float rotation_offset[3], rotation_pivot[3], scaling_offset[3], scaling_pivot[3];
} fyx_transform_statics;
int32_t fyx_set_local_trs(fyx_ctx *ctx, uint32_t count, const uint32_t *idx, const fyx_trs *trs);
/* Transform::set_rotation only (what skeletal animation does to most bones every frame): 16 B per node; position and
 * scale stay what the node's last fyx_set_local_trs sent (identity for a node that never got one). */
int32_t fyx_set_local_rotations(fyx_ctx *ctx, uint32_t count, const uint32_t *idx, const float *quat_ijkw);
int32_t fyx_set_transform_statics(fyx_ctx *ctx, uint32_t count, const uint32_t *idx, const fyx_transform_statics *statics);
/* Base::set_visibility / set_enabled / frustum_culling / cast_shadows (VisibilityChanged / EnabledFlagChanged). */
int32_t fyx_set_flags(fyx_ctx *ctx, uint32_t count, const uint32_t *idx, const uint32_t *flags);
int32_t fyx_set_render_masks(fyx_ctx *ctx, uint32_t count, const uint32_t *idx, const uint32_t *render_mask);
int32_t fyx_set_local_aabbs(fyx_ctx *ctx, uint32_t count, const uint32_t *idx, const float *aabb_minmax);

/* One skinned Surface of Mesh node `mesh_node` (scene/mesh/surface.rs:1249-1271): `bone_nodes` = Surface::bones
 * indices (≤255), inv_bind_m16 = each bone's Base::inv_bind_pose_transform (scene/base.rs:482), verts = the
 * surface's VertexBuffer bytes (n_verts * layout->stride).  Surfaces of one mesh are folded into its world
 * AABB in call order (scene/mesh/mod.rs:676-682).  verts may be NULL with n_verts 0 (palette only). */
int32_t fyx_add_skinned_surface(fyx_ctx *ctx, uint32_t mesh_node, uint32_t n_bones, const uint32_t *bone_nodes,
                                const float *inv_bind_m16, uint32_t n_verts, const void *verts,
                                const fyx_vertex_layout *layout, uint32_t *out_surface_id);
/* Optional: size the device-side bone / vertex tables once for `total_bones` palette entries and
 * `total_verts` vertices (sum over all surfaces to be added) instead of growing them on demand. */
int32_t fyx_reserve_skinning(fyx_ctx *ctx, uint64_t total_bones, uint64_t total_verts);
/* Finish a batch of fyx_add_skinned_surface calls (builds the device-side bone/vertex tables). Called
 * implicitly by the first per-frame call that needs them. */
int32_t fyx_commit_surfaces(fyx_ctx *ctx);

/* ---- per frame ----------------------------------------------------------------------------- */
/* Graph::update → process_node_messages (scene/graph/mod.rs:1303-1399, 1459-1473): global transforms
 * (update_global_transform_recursively :1199-1241), global visibility / enabled (:1166-1197), world AABBs
 * (AxisAlignedBoundingBox::transform, fyrox-math/src/aabb.rs:264-287; Mesh::on_global_transform_changed,
 * scene/mesh/mod.rs:667-689). */
int32_t fyx_update_transforms(fyx_ctx *ctx, uint32_t update_flags);

/* RenderDataBundleStorage::from_graph reduced to its visible-node set (renderer/bundle.rs:873-1009):
 * for each frustum f, the nodes for which NodeTrait::should_be_rendered(frustum, cam_mask[f])
 * (scene/node/mod.rs:231-256, Frustum::is_intersects_aabb fyrox-math/src/frustum.rs:222-245) holds, that are
 * alive, renderable and reachable from the root, and (pass_flags[f] & FYX_PASS_SHADOW) ⇒ cast_shadows.
 * cam_mask NULL = all ones; pass_flags NULL = 0.  The list is a SET: its order is unspecified. */
int32_t fyx_cull(fyx_ctx *ctx, uint32_t n_frusta, const fyx_frustum *frusta, const uint32_t *cam_mask,
                 const uint32_t *pass_flags);
/* fyx_update_transforms + fyx_cull in one pass over the node arrays (world AABBs stay in registers). */
int32_t fyx_update_and_cull(fyx_ctx *ctx, uint32_t update_flags, uint32_t n_frusta, const fyx_frustum *frusta,
                            const uint32_t *cam_mask, const uint32_t *pass_flags);
/* Visible list of frustum f as node indices (global_index values): host copy (pinned) ... */
int32_t fyx_get_visible(fyx_ctx *ctx, uint32_t frustum, const uint32_t **out_idx, uint32_t *out_count);
/* ... or device-resident (for a GPU consumer / a collective); *d_count points at one device u32. */
int32_t fyx_get_visible_device(fyx_ctx *ctx, uint32_t frustum, const uint32_t **d_idx, const uint32_t **d_count);

/* N4 (light list) — the `collect_lights` part of RenderDataBundleStorage::from_graph (renderer/bundle.rs:926-974): for
 * every frustum of the most recent cull, the FYX_NODE_LIGHT nodes whose world bounding box the frustum intersects and
 * that are globally visible and enabled (no reachability / render-mask / frustum_culling-flag test, as in the
 * reference).  Lists come back in ascending node index = the reference's pool order.  Lights in sub-trees detached from
 * the root are outside the contract: the reference never updates such sub-trees, this library updates every tree. */
int32_t fyx_cull_lights(fyx_ctx *ctx);
/* The reflection-probe part of the same loop (renderer/bundle.rs:918-925): per observer of fyx_set_observers the LAST node in pool
 * order that carries FYX_NODE_REFLECTION_PROBE and whose world bounding box contains the observer's translation (inclusive) —
 * `storage.environment_map`; FYX_NONE = none.  out_probe receives one node index per observer. */
int32_t fyx_select_reflection_probes(fyx_ctx *ctx, uint32_t count, uint32_t *out_probe);
int32_t fyx_get_visible_lights(fyx_ctx *ctx, uint32_t frustum, const uint32_t **out_idx, uint32_t *out_count);

/* N4 (shadow casters) — the shadow-map loop of the deferred light renderer (renderer/light.rs:509-606, 695-763) with the
 * per-map cull of the spot and point shadow renderers (renderer/shadow/spot.rs:142, shadow/point.rs:162-180), on the device.
 *
 * fyx_set_light_sources: the LightSource data of `count` light nodes (idx NULL = nodes 0..count-1) that the world
 * transform does not give: kind, SpotLight::full_cone_angle (spot only) and SpotLight::distance / PointLight::radius.
 * FYX_LIGHT_UNKNOWN removes the node's record.  fyx_set_topology keeps a record with its node index while the node is alive
 * before and after the call; any other node index starts again without a record.  The projection's
 * one transcendental, m22 = 1 / tan(fovy / 2) (fovy = full_cone_angle, or FRAC_PI_2 for a point light), is evaluated here
 * with the platform's tanf; everything the device does with the record is + − × ÷ √.
 *
 * fyx_cull_shadow_casters: takes frustum `camera_frustum` of the most recent cull as the camera (its planes and its
 * cam_mask = observer.render_mask) and `camera_translation` as observer.position.translation, and produces every shadow
 * map the reference renders for that camera, in its order: lights in pool order, 1 map per spot light, 6 per point
 * light in CubeMapFaceDescriptor::cube_faces() order.  A light gets maps only when it is in the camera's light list
 * (fyx_cull_lights' rule), its node has FYX_NODE_CAST_SHADOWS, distance_to_camera <= {spot,point}_shadows_distance,
 * shadows are enabled for its kind, and the camera frustum intersects the sphere (position, light_radius), light_radius =
 * max(local scale) * distance_or_radius with the scale of the node's last TRS record (identity without one).  Each map
 * gets the cascade index of light.rs:592-606, view_projection = P · V (spot: look_at_rh(pos, pos − up, look); point:
 * look_at_rh(pos, pos + face.look, face.up); z_near 0.01, z_far light_radius) and the visible set of
 * from_graph(map frustum, cam_mask, shadow pass): alive, renderable, reachable, should_be_rendered and cast_shadows.
 * One pass over the nodes tests every map; list memory grows with the visible entries.  Synchronous.
 * Directional lights get maps only through fyx_cull_shadow_casters_csm (below); fyx_cull_shadow_casters(..) is exactly
 * fyx_cull_shadow_casters_csm(.., NULL).  Not modelled: light occlusion queries (use_light_occlusion_culling = false),
 * shadow alpha, cascade distances, shadow bias and other shading-only values.  The lists' instances: made with
 * fyx_enable_instances, the cull also records each entry's slot for fyx_pack_shadow_instances.
 * Returns FYX_ERR_STATE when no cull has been made, a frame is still in flight, LOD ranges with observers are active or a
 * node carries FYX_NODE_STATIC_BATCH (the per-map LOD filter and static-batch pruning are not modelled: the call refuses
 * rather than give a different set), or the context is sharded (fyx_comm_init); FYX_ERR_INVALID_ARGUMENT when
 * camera_frustum is not a frustum of the last cull.
 *
 * fyx_set_csm_options: the FrustumSplitOptions (scene/light/directional.rs:60-91) of `count` directional light nodes (idx
 * NULL = nodes 0..count-1).  A node without a record uses the reference's default, Absolute {5, 25, 64}.  fyx_set_topology
 * keeps a record with its node index while the node is alive before and after the call; any other node index starts again
 * from the default.  FYX_ERR_INVALID_ARGUMENT for a node out of range or `relative` other than 0 / 1.
 *
 * fyx_cull_shadow_casters_csm: fyx_cull_shadow_casters plus the cascaded shadow maps of the directional lights
 * (renderer/shadow/csm.rs:165-277).  A directional light in the camera's light list gets maps when its node has
 * FYX_NODE_CAST_SHADOWS, cam->csm_enabled is set and the camera frustum intersects the sphere (position, max(local scale)
 * * f32::MAX) (light.rs:555-565); it then gets three maps in the light loop's pool order, face 0, cascade 0, 1, 2.  Cascade
 * i splits the camera's depth range at z_values = [z_near, splits[0..3]] (Absolute) or [z_near, z_far * splits[k]]
 * (Relative), builds the camera projection of that slice (scene/camera.rs:89-174) and its frustum (Frustum::default if
 * it has none), and takes view_projection = new_orthographic(box) · look_at_lh(center − up/|up|, center, look/|look|), the box being
 * the slice's corners in light space with its depth stretched ×10.  Its list is from_graph(map frustum, cam_mask, shadow
 * pass), as for the spot and point maps; fyx_pack_shadow_instances sorts its instances by the map's look_at_lh.  The
 * perspective's 1 / tan(fov / 2) is evaluated here with the platform's tanf.  cam NULL or csm_enabled = 0: directional
 * lights get no maps.  Same refusals as fyx_cull_shadow_casters, plus FYX_ERR_INVALID_ARGUMENT for an unknown projection
 * kind.  Inputs for which the reference panics (superimposed planes, a collapsed light-space box) give a defined result.
 *
 * fyx_cull_shadow_casters_pruned: fyx_cull_shadow_casters_csm (same parameters, same map table: the same maps in the same
 * order, view_projection bit for bit) where every map's list is from_graph with that map's own LOD filter and static-batch
 * pruning, as the reference builds one RenderDataBundleStorage per map (renderer/bundle.rs:873-1009):
 *   - LOD filter: the ranges of fyx_set_lod_ranges, whenever any node has one (fyx_set_observers takes no part: it
 *     describes the frusta of fyx_cull).  The map's observer is the light's global position with z_near 0.01 and z_far
 *     light_radius for a spot map and each cube face of a point light (light.rs:700-728, shadow/point.rs:162-190), and for
 *     cascade i the look_at_lh eye center + light_direction with the slice's z_near and guarded z_far (shadow/csm.rs:195-270).
 *     A LOD object whose normalised distance (dist − z_near) / (z_far − z_near) lies outside its [begin, end] hides itself
 *     and its whole sub-tree in that map only.
 *   - Static batches: an FYX_NODE_STATIC_BATCH node that is in a map's list (frustum, camera mask, cast_shadows) hides its
 *     sub-tree in that map (Mesh::collect_render_data's Break, scene/mesh/mod.rs:691-725); where it is not in the list its
 *     children are visited as usual.
 * A static batch's shadow instance carries the identity world matrix (fyx_pack_shadow_instances), as on the camera path.
 * The per-map state grows with the pruners (LOD objects and static batches), not with nodes x maps: one u32 per slot (the
 * nearest pruner on the node's path, rebuilt by the first pruned cull after fyx_set_topology, fyx_set_lod_ranges or a
 * fyx_set_flags that changes an FYX_NODE_STATIC_BATCH bit) and two rows of ceil(maps / 32) words per pruner.  On a context
 * with no LOD range and no static batch it runs exactly the kernels of fyx_cull_shadow_casters_csm; fyx_cull_shadow_casters_csm
 * equals fyx_cull_shadow_casters_pruned on such a context and refuses (FYX_ERR_STATE) on any other.  Refusals otherwise as
 * fyx_cull_shadow_casters_csm; FYX_ERR_OUT_OF_MEMORY when the pruner table does not fit. */
#define FYX_LIGHT_UNKNOWN 0u
#define FYX_LIGHT_SPOT 1u
#define FYX_LIGHT_POINT 2u
#define FYX_LIGHT_DIRECTIONAL 3u
typedef struct fyx_light_source {
    uint32_t kind;             /* FYX_LIGHT_* */
    float full_cone_angle;     /* radians, spot lights only */
    float distance_or_radius;  /* SpotLight::distance or PointLight::radius */
} fyx_light_source;
typedef struct fyx_shadow_settings { /* QualitySettings, renderer/settings.rs:112-191 */
    float spot_shadows_distance;
    float point_shadows_distance;
    uint32_t spot_shadows_enabled;
    uint32_t point_shadows_enabled;
} fyx_shadow_settings;
typedef struct fyx_shadow_map {
    uint32_t light;            /* light node index */
    uint32_t face;             /* 0 for a spot light, the cube face 0..5 for a point light */
    uint32_t cascade;          /* 0, 1 or 2 */
    uint32_t first, count;     /* the map's visible list is entries[first, first + count), order unspecified */
    float view_projection[16]; /* column-major */
} fyx_shadow_map;
int32_t fyx_set_light_sources(fyx_ctx *ctx, uint32_t count, const uint32_t *idx, const fyx_light_source *src);
int32_t fyx_cull_shadow_casters(fyx_ctx *ctx, uint32_t camera_frustum, const float camera_translation[3], const fyx_shadow_settings *settings);
#define FYX_PROJECTION_PERSPECTIVE 0u
#define FYX_PROJECTION_ORTHOGRAPHIC 1u
typedef struct fyx_csm_options { /* FrustumSplitOptions */
    uint32_t relative;           /* 0: Absolute { far_planes }, 1: Relative { fractions } */
    float splits[3];
} fyx_csm_options;
typedef struct fyx_csm_camera {
    uint32_t projection;         /* FYX_PROJECTION_* */
    float fov_or_vertical_size;  /* PerspectiveProjection::fov (radians) or OrthographicProjection::vertical_size */
    float z_near, z_far;         /* the projection's own values (ObserverPosition::from_camera, renderer/observer.rs:64-72) */
    float frame_size[2];         /* the frame the cascades are rendered for: the G-buffer's width and height (light.rs:767) */
    float view_matrix[16];       /* Camera::view_matrix, column-major */
    uint32_t csm_enabled;        /* QualitySettings::csm_settings.enabled */
} fyx_csm_camera;
int32_t fyx_set_csm_options(fyx_ctx *ctx, uint32_t count, const uint32_t *idx, const fyx_csm_options *opts);
int32_t fyx_cull_shadow_casters_csm(fyx_ctx *ctx, uint32_t camera_frustum, const float camera_translation[3], const fyx_shadow_settings *settings,
                                    const fyx_csm_camera *cam);
int32_t fyx_cull_shadow_casters_pruned(fyx_ctx *ctx, uint32_t camera_frustum, const float camera_translation[3],
                                       const fyx_shadow_settings *settings, const fyx_csm_camera *cam /* NULL = no cascades */);
/* Result of the last fyx_cull_shadow_casters: pinned host copies ... */
int32_t fyx_get_shadow_maps(fyx_ctx *ctx, const fyx_shadow_map **out_maps, uint32_t *out_n_maps, const uint32_t **out_entries);
/* ... or the device arrays (*out_n_maps is a host value). */
int32_t fyx_get_shadow_maps_device(fyx_ctx *ctx, const fyx_shadow_map **d_maps, uint32_t *out_n_maps, const uint32_t **d_entries);

/* N4 (LOD filter) — the lod_filter of RenderDataBundleStorage::from_graph (renderer/bundle.rs:898-916, 988-1004): a node
 * that is an object of a LOD level is visible for an observer only while its normalised distance
 * (|observer.translation − global_position| − z_near) / (z_far − z_near) lies in the level's [begin, end]; a node that is
 * filtered out hides its whole sub-tree (the DFS does not descend).
 * fyx_set_lod_ranges: per LOD object the range of the level it belongs to (2 floats each: begin, end; begin = NaN removes
 * the node from LOD control).  The host resolves "listed in several levels" the way the reference's loop does — owners in
 * pool order, levels and objects in order, the last write wins.  Carried over by fyx_set_topology with the node indices.
 * fyx_set_observers: ObserverPosition::{translation, z_near, z_far} of the frusta of the culls that follow, one per
 * frustum (count 0 = no LOD filtering).  While both are set the cull runs un-fused: update, then one small pass per
 * hierarchy level that holds LOD objects or static batches, over those nodes only, that propagates the filter bits from
 * parents to children, then the cull over all nodes. */
typedef struct fyx_observer {
    float translation[3];
    float z_near, z_far;
} fyx_observer;
int32_t fyx_set_lod_ranges(fyx_ctx *ctx, uint32_t count, const uint32_t *idx, const float *begin_end);
int32_t fyx_set_observers(fyx_ctx *ctx, uint32_t count, const fyx_observer *observers);

/* N4 (scene observers) — ObserversCollection::from_scene (renderer/observer.rs:88-153) and one from_graph per observer
 * (renderer/mod.rs:1034-1047, 1364-1400), on the device, in one call.
 *
 * fyx_set_cameras / fyx_set_reflection_probes: the Camera / ReflectionProbe data of `count` nodes (idx NULL = nodes
 * 0..count-1) that the global transform does not give.  A record with projection FYX_PROJECTION_NONE (camera) or present 0
 * (probe) removes the node's record.  Records are kept by node index: fyx_set_topology keeps a record while the node is
 * alive before and after the call; any other node index starts again without a record.  The perspective's one transcendental, 1 / tan(fov / 2), is evaluated here with the
 * platform's tanf (a probe's fov is 90f32.to_radians() = FRAC_PI_2, the point lights' value).  Setting a probe's record
 * makes it due, as does fyx_force_reflection_probe_update (ReflectionProbe::force_update, scene/probe.rs:215-218).
 *
 * fyx_cull_scene_observers: the observers of the scene, in the reference's order — first the six faces of every due
 * reflection probe (probes in pool order, faces in CubeMapFaceDescriptor::cube_faces() order), then every camera in pool
 * order — each with its matrices, its visible list, its light list and its environment map.
 *   - A node counts when it is alive and FYX_NODE_GLOBAL_ENABLED after the last update (observer.rs:91); a camera also
 *     needs `enabled`.  A probe is due when its mode is FYX_PROBE_UPDATE_EACH_FRAME, or when it has not been emitted since
 *     its record was set or its update forced (probe.rs:276-290, observer.rs:99-102); every call that emits a probe and
 *     succeeds marks it rendered (a call that fails leaves it due).  That bit lives on the device and survives fyx_set_topology.
 *   - Camera (scene/camera.rs:454-462, observer.rs:64-74): view = look_at_rh(pos, pos + look, up) with the global
 *     matrix's translation, column 2 and column 1 as they are (not normalised); projection = Projection::matrix(frame
 *     size) with its guards (camera.rs:89-173), the frame size being the record's when it is not 0,0 (a render target),
 *     else the call's; translation = the global position, z_near / z_far the record's raw values.
 *   - Probe face (observer.rs:104-145): translation = global position + rendering_position; projection = the guarded
 *     perspective of fov FRAC_PI_2 and aspect 1; view = look_at_rh(t, t + face.look, face.up).
 *   - Frustum: from_view_projection_matrix(projection · view).unwrap_or_default() (renderer/bundle.rs:893-896).
 *   - Visible list: from_graph without the shadow pass: alive, renderable, reachable, should_be_rendered with the node's
 *     render mask against the observer's (render_mask = the camera's or probe's node mask), the LOD filter of
 *     fyx_set_lod_ranges with the observer's translation and z range, and static-batch Break (scene/mesh/mod.rs:691-725)
 *     — always honoured.  Order inside a list is unspecified.
 *   - Light list: fyx_cull_lights' rule for the observer's frustum, in pool order.  Environment map: for a camera
 *     fyx_select_reflection_probes' rule for its translation; FYX_NONE for a probe face (renderer/mod.rs:1045-1047).
 * One pass over the nodes counts every observer's list; the call is synchronous.  FYX_ERR_STATE on a sharded context, while
 * a frame is in flight, or before fyx_set_topology; FYX_ERR_INVALID_ARGUMENT for a NULL or non-positive frame_size.
 * fyx_set_* return FYX_ERR_INVALID_ARGUMENT for an unknown projection kind or update mode or a node out of range. */
#define FYX_PROJECTION_NONE 0xFFFFFFFFu
typedef struct fyx_camera {             /* Camera fields, scene/camera.rs */
    uint32_t enabled;                   /* Camera::is_enabled */
    uint32_t projection;                /* FYX_PROJECTION_PERSPECTIVE / _ORTHOGRAPHIC; FYX_PROJECTION_NONE removes the record */
    float fov_or_vertical_size;         /* PerspectiveProjection::fov (radians) or OrthographicProjection::vertical_size */
    float z_near, z_far;                /* the projection's own values */
    float frame_size[2];                /* the render target's size (camera.rs:813-826); 0,0 = the call's frame size */
} fyx_camera;
int32_t fyx_set_cameras(fyx_ctx *ctx, uint32_t count, const uint32_t *idx, const fyx_camera *cameras);
#define FYX_PROBE_UPDATE_ONCE 0u
#define FYX_PROBE_UPDATE_EACH_FRAME 1u
typedef struct fyx_reflection_probe {   /* ReflectionProbe fields, scene/probe.rs */
    uint32_t present;                   /* 0 removes the record */
    uint32_t update_mode;               /* FYX_PROBE_UPDATE_* */
    float z_near, z_far;
    float rendering_position[3];        /* added to the global position: global_rendering_position, probe.rs:221-223 */
} fyx_reflection_probe;
int32_t fyx_set_reflection_probes(fyx_ctx *ctx, uint32_t count, const uint32_t *idx, const fyx_reflection_probe *probes);
int32_t fyx_force_reflection_probe_update(fyx_ctx *ctx, uint32_t count, const uint32_t *idx);
#define FYX_OBSERVER_PROBE_FACE 0u
#define FYX_OBSERVER_CAMERA 1u
typedef struct fyx_scene_observer {
    uint32_t node, kind, face;          /* FYX_OBSERVER_PROBE_FACE (face 0..5) or FYX_OBSERVER_CAMERA (face 0) */
    uint32_t render_mask;               /* Observer::render_mask: the node's render mask */
    uint32_t first, count;              /* visible list: entries[first, first + count), order unspecified */
    uint32_t lights_first, lights_count;/* light list: light_entries[lights_first, + lights_count), ascending node index */
    uint32_t environment_map;           /* reflection-probe node, FYX_NONE = none */
    float translation[3], z_near, z_far;/* ObserverPosition */
    float view[16], projection[16], view_projection[16]; /* column-major */
} fyx_scene_observer;
int32_t fyx_cull_scene_observers(fyx_ctx *ctx, const float frame_size[2]);
/* Result of the last fyx_cull_scene_observers: pinned host copies, valid until the next call ... */
int32_t fyx_get_scene_observers(fyx_ctx *ctx, const fyx_scene_observer **out_table, uint32_t *out_n, const uint32_t **out_entries,
                                const uint32_t **out_light_entries);
/* ... or the device arrays (*out_n is a host value). */
int32_t fyx_get_scene_observers_device(fyx_ctx *ctx, const fyx_scene_observer **d_table, uint32_t *out_n, const uint32_t **d_entries,
                                       const uint32_t **d_light_entries);
/* Instances of the observers: fyx_pack_scene_observer_instances, below with the shadow maps' pack.
 *
 * fyx_cull_scene_shadow_casters: the shadow maps every observer of the last successful fyx_cull_scene_observers renders
 * (render_scene_observer runs the deferred light renderer for each observer, probe faces included: renderer/mod.rs:964-1120,
 * renderer/light.rs:509-782), and their lists, in one call.
 *   - For every observer in table order and every light of its light list (pool order), the gates of
 *     fyx_cull_shadow_casters_csm with the observer as the camera: a light with no fyx_set_light_sources record is skipped
 *     (Unknown); cast_shadows; the distance gate against the observer's translation; is_intersects_sphere against its
 *     frustum; the cascade index from that distance; directional lights need csm_enabled.
 *   - A directional light's three cascades take the observer's projection kind, 1 / tan(fov / 2) or vertical size (for a
 *     probe face the FRAC_PI_2 value), raw z_near / z_far, view matrix, and frame size: for a camera its render target's
 *     size when it is not 0,0, else the frame size of that fyx_cull_scene_observers call; for a probe face aspect 1 (a cube
 *     face is square; Projection::matrix uses only w / h, camera.rs:89-106).
 *   - Every map carries its observer's render_mask: a node is in a map's list when it passes the shadow pass (cast_shadows),
 *     that mask and the map's frustum.  Each map's LOD filter (its own observer: the light's position, 0.01 and the radius
 *     for spot and point maps; the look_at_lh eye and the slice's depths for cascades) and static-batch Break (with the
 *     map's mask) are always honoured, as in fyx_cull_shadow_casters_pruned.
 *   - Spot and point maps with equal (light, face, cascade, render mask) are one row of the map table, culled and listed
 *     once: their frustum, LOD observer and list do not depend on the observer (light.rs:700-728, shadow/point.rs:162-190).
 *     Cascades are never shared.  Rows are numbered in order of first reference, and every field of a row holds for every
 *     observer that references it.
 *   - The refs list every (observer, map) pair in the reference's render order: observers in table order, then lights in
 *     list order, then faces 0..5 or cascades 0..2.
 * The result replaces the last shadow cull's: fyx_get_shadow_maps[_device], fyx_pack_shadow_instances, the shadow instance
 * getters and fyx_pack_shadow_bone_matrices work on its map table unchanged; a later fyx_cull_shadow_casters* makes
 * fyx_get_scene_shadow_maps return FYX_ERR_STATE.  The call is synchronous.  FYX_ERR_INVALID_ARGUMENT for a NULL ctx or
 * settings; FYX_ERR_STATE before a successful fyx_cull_scene_observers, after fyx_set_topology or any hierarchy update
 * since that call (its table describes another frame), on a sharded context, or while a frame is in flight. */
typedef struct fyx_scene_shadow_map {   /* one shadow map an observer renders */
    uint32_t observer;                  /* row of the last fyx_cull_scene_observers table */
    uint32_t map;                       /* row of fyx_get_shadow_maps' table: light, face, cascade, list, view_projection */
} fyx_scene_shadow_map;
int32_t fyx_cull_scene_shadow_casters(fyx_ctx *ctx, const fyx_shadow_settings *settings, uint32_t csm_enabled);
/* The refs of the last fyx_cull_scene_shadow_casters: a pinned host copy, valid until the next call ... */
int32_t fyx_get_scene_shadow_maps(fyx_ctx *ctx, const fyx_scene_shadow_map **out_refs, uint32_t *out_n);
/* ... or the device array (*out_n is a host value). */
int32_t fyx_get_scene_shadow_maps_device(fyx_ctx *ctx, const fyx_scene_shadow_map **d_refs, uint32_t *out_n);

/* ---- N4: blend shapes (morph targets) ahead of the skinning ------------------------------------------------ */
/* The standard shader adds, for every blend shape i of the surface in order, offsets.position * weight to the vertex
 * position and offsets.normal * weight to the normal BEFORE skinning (fyrox-material/src/shader/standard/opengl/
 * standard.shader:167-173), weight = BlendShape::weight / 100 (scene/mesh/mod.rs:794-798).  `records` is the content of
 * BlendShapesContainer::blend_shape_storage as from_lists builds it (scene/mesh/surface.rs:92-218): n_shapes layers of
 * layer_stride (= width * height >= n_verts) records of 9 binary16 values — position, normal, tangent offsets of vertex
 * v at record v of the layer (tangents are not part of the skinned streams and are ignored).  `weights` = the
 * BlendShape::weight values (0..100), NULL = 100 each (BlendShape::default()).  n_shapes = 0 removes them.
 * Costs 12 more bytes read per vertex and shape in fyx_skin; surfaces without shapes are unaffected. */
#define FYX_MAX_BLEND_SHAPES 128u /* ShaderDefinition::MAX_BLEND_SHAPE_WEIGHT_GROUPS * 4, fyrox-material/src/shader/mod.rs:616 */
int32_t fyx_set_blend_shapes(fyx_ctx *ctx, uint32_t surface_id, uint32_t n_shapes, const void *records, uint32_t layer_stride,
                             const float *weights);
int32_t fyx_set_blend_shape_weights(fyx_ctx *ctx, uint32_t surface_id, uint32_t n, const float *weights);

/* SurfaceInstanceData::bone_matrices for every skinned surface (scene/mesh/mod.rs:781-793):
 * P[k] = bone_k.global_transform * bone_k.inv_bind_pose_transform; dead / FYX_NONE bone ⇒ identity. */
int32_t fyx_build_palettes(fyx_ctx *ctx);
/* Linear-blend skinning of every skinned surface: positions as Mesh::accurate_world_bounding_box
 * (scene/mesh/mod.rs:501-522), normals as the standard shader (fyrox-material/src/shader/standard/opengl/
 * standard.shader:192-195) — into device-resident position / normal streams. */
int32_t fyx_skin(fyx_ctx *ctx);

/* One whole frame of render prep, in stream order, with one host synchronisation at the end:
 * upload changed local matrices → update (+cull) → palettes → skin → visible lists to the host.
 * Any of the parts may be empty (count 0 / n_frusta 0 / no surfaces). */
typedef struct fyx_frame_desc {
    uint32_t struct_size;
    uint32_t update_flags;
    uint32_t n_changed;            /* changed local matrices this frame */
    const uint32_t *changed_idx;   /* NULL = nodes 0..n_changed-1 */
    const float *changed_m16;      /* n_changed * 16 f32 ... */
    const fyx_trs *changed_trs;    /* ... or, if non-NULL, n_changed fyx_trs records (changed_m16 ignored) */
    const float *changed_rot;      /* ... or, if non-NULL, n_changed rotations (4 f32 each; the others ignored) */
    uint32_t n_frusta;
    const fyx_frustum *frusta;
    const uint32_t *cam_mask;
    const uint32_t *pass_flags;
    uint32_t do_palettes;
    uint32_t do_skin;
    uint32_t readback_visible;     /* copy counts + lists to the host before returning */
    uint32_t flags;                /* FYX_FRAME_* */
    /* since ABI 2 (struct_size tells which fields the caller has): */
    uint32_t do_animate;           /* first run fyx_animate(animate_dt): AnimationPlayer::update before Graph::update */
    float animate_dt;
} fyx_frame_desc;
/* Do not synchronise with the host at the end of fyx_render_prep: the frame is only enqueued.  Inputs must
 * stay untouched until the frame is waited for (fyx_frame_wait / fyx_sync).  Pinned inputs are uploaded on
 * a copy stream into alternating staging buffers, so the upload of frame i+1 overlaps the kernels of
 * frame i.  With readback_visible the read-back is deferred: at most two such frames may be in flight,
 * fyx_frame_wait collects the oldest one and makes its visible lists the ones fyx_get_visible returns. */
#define FYX_FRAME_ASYNC (1u << 0)
/* Multi-GPU (after fyx_comm_init): all-gather the frame's visible lists as soon as the cull is done, on a
 * separate stream, overlapped with the palette / skinning kernels of the same frame; the frame is complete
 * when the gathered lists are (fyx_get_visible_gathered*).  Collective: every rank issues the frame.
 * With readback_visible every rank also copies its OWN lists into the node-wide host segment (one PCIe link per rank);
 * fyx_get_visible_gathered on any rank then returns the whole lists from that segment and fyx_get_visible the rank's
 * own part of it (fyx_comm_mode tells whether the segment is in use; without it the host copy comes from the rank's
 * device). */
#define FYX_FRAME_ALLGATHER (1u << 1)
/* With FYX_FRAME_ALLGATHER on a pipelined (async + read-back) frame and NO host segment (FYX_HOSTSEG=0 or not available):
 * bring only THIS rank's lists to the host (fyx_get_visible); the gathered lists stay device-resident.  One process of the
 * job — the one that feeds the CPU-side renderer — leaves it off and receives the whole lists through its pinned copy; the
 * others do not multiply that PCIe traffic by the number of GPUs.  With the host segment the flag changes nothing: every
 * rank copies its own lists only. */
#define FYX_FRAME_READBACK_OWN (1u << 2)
int32_t fyx_frame_wait(fyx_ctx *ctx);
int32_t fyx_render_prep(fyx_ctx *ctx, const fyx_frame_desc *frame);

/* ---- read-back (tests, tools, and the parts of the engine that stay on the CPU) -------------- */
int32_t fyx_get_global_matrices(fyx_ctx *ctx, uint32_t count, const uint32_t *idx, float *out_m16);   /* Base::global_transform */
int32_t fyx_get_world_aabbs(fyx_ctx *ctx, uint32_t count, const uint32_t *idx, float *out_minmax);    /* NodeTrait::world_bounding_box */
int32_t fyx_get_global_flags(fyx_ctx *ctx, uint32_t count, const uint32_t *idx, uint32_t *out_flags);
int32_t fyx_get_palette(fyx_ctx *ctx, uint32_t surface_id, float *out_m16 /* n_bones*16 */);
int32_t fyx_get_skinned(fyx_ctx *ctx, uint32_t surface_id, float *out_pos3, float *out_nrm3 /* n_verts*3 each; either may be NULL */);
int32_t fyx_get_skinned_device(fyx_ctx *ctx, uint32_t surface_id, const float **d_pos3, const float **d_nrm3);
int32_t fyx_get_timings(fyx_ctx *ctx, fyx_timings *out);
/* Number of kernels this context has launched so far (bench.py's gpu_launches). */
uint64_t fyx_kernel_launch_count(const fyx_ctx *ctx);

/* ---- N2: animation sampling on the device (SURVEY §8f) ---------------------------------------- */
/* What AnimationPlayer nodes do on the CPU before Graph::update (scene/animation/mod.rs:83-88,340-346): every
 * enabled animation ticks — its tracks' curves are sampled at the current time position (fyrox-animation/src/
 * lib.rs:895-914, container.rs:162-301, fyrox-math/src/curve.rs:252-309), the pose is applied to the target
 * nodes' position / rotation / scale (scene/animation/mod.rs:147-179) and the time position advances
 * (lib.rs:471-496, 432-440).  With the curves resident in HBM nothing is uploaded per frame.
 * Properties no track writes keep the value of the node's last fyx_set_local_trs record (identity if none);
 * pivots / offsets / pre- and post-rotation come from fyx_set_transform_statics.
 * Parity: Vector3 and UnitQuaternion tracks bit-exact; UnitQuaternionEuler tracks use sin/cos (platform libm in the
 * reference): ~1e-7 absolute on the quaternion.  Signals, root motion, property bindings and the blend-machine
 * (ABSM) layers are not modelled. */
#define FYX_KEY_CONSTANT 0u /* CurveKeyKind (fyrox-math/src/curve.rs:33-45) */
#define FYX_KEY_LINEAR 1u
#define FYX_KEY_CUBIC 2u
typedef struct fyx_curve_key {
    float location, value;
    uint32_t kind;                     /* FYX_KEY_* */
    float left_tangent, right_tangent; /* tan(angle), Cubic only */
} fyx_curve_key;

#define FYX_TV_REAL 0u /* TrackValueKind (fyrox-animation/src/container.rs:41-54) */
#define FYX_TV_VECTOR2 1u
#define FYX_TV_VECTOR3 2u
#define FYX_TV_VECTOR4 3u
#define FYX_TV_QUAT_EULER 4u
#define FYX_TV_QUAT 5u
#define FYX_BIND_POSITION 0u /* ValueBinding (fyrox-animation/src/value.rs:358-374) */
#define FYX_BIND_SCALE 1u
#define FYX_BIND_ROTATION 2u
typedef struct fyx_anim_track {
    uint32_t target_node;  /* TrackBinding::target (node index) */
    uint32_t binding;      /* FYX_BIND_* */
    uint32_t value_kind;   /* FYX_TV_* */
    uint32_t enabled;      /* TrackBinding::enabled */
    uint32_t n_curves;     /* TrackDataContainer::curves.len(): fewer than the kind needs = fetch returns None */
    uint32_t first_key[4]; /* curve c = keys[first_key[c] .. first_key[c] + n_keys[c]), sorted by location */
    uint32_t n_keys[4];
} fyx_anim_track;

typedef struct fyx_animation_desc {
    uint32_t struct_size;
    uint32_t n_tracks;
    const fyx_anim_track *tracks; /* in AnimationTracksData::tracks order */
    uint32_t n_keys;
    const fyx_curve_key *keys;
    float speed;                  /* Animation defaults (lib.rs:922-945): 1.0 */
    float time_position;
    float time_slice_start, time_slice_end;
    uint32_t looped;
    uint32_t enabled;
} fyx_animation_desc;

/* Add an animation; ids are 0,1,2,... in call order = the order update_animations walks them. */
int32_t fyx_anim_add(fyx_ctx *ctx, const fyx_animation_desc *desc, uint32_t *out_id);
int32_t fyx_anim_clear(fyx_ctx *ctx);
int32_t fyx_anim_set_enabled(fyx_ctx *ctx, uint32_t anim, uint32_t enabled);                        /* Animation::set_enabled */
int32_t fyx_anim_set_track_enabled(fyx_ctx *ctx, uint32_t anim, uint32_t track, uint32_t enabled);  /* TrackBinding::set_enabled */
int32_t fyx_anim_set_speed(fyx_ctx *ctx, uint32_t anim, float speed);
int32_t fyx_anim_set_time_position(fyx_ctx *ctx, uint32_t anim, float time); /* wraps / clamps into the time slice (lib.rs:432-440) */
int32_t fyx_anim_get_time_positions(fyx_ctx *ctx, uint32_t first, uint32_t count, float *out);
/* Pose blending, the smallest useful subset of the blend machine (fyrox-animation/src/machine): the listed animations
 * stop being applied directly (AnimationPlayer::auto_apply = false) and become, in this order, the PlayAnimation sources
 * of ONE PoseNode::BlendAnimations with constant weights (machine/node/blend.rs:136-166) in a one-layer, one-state
 * machine: every enabled source still ticks (machine/mod.rs:366-372; a disabled one keeps contributing the pose of its
 * last tick), the output pose takes a clone of the first source that has values for a node and blends every later
 * source into it per binding — AnimationPose::blend_with / TrackValue::blend_with (pose.rs:41-101, value.rs:201-227:
 * nalgebra lerp for vectors, shortest-way nlerp for rotations) — and is then applied.  Groups are applied after the
 * directly applied animations, in creation order.  Restrictions: Vector3 / UnitQuaternion(Euler) tracks only, one track
 * per (node, property) and animation, an animation in at most one group.  Transitions, parameters, masks, blend
 * spaces, layers > 1: not modelled. */
int32_t fyx_anim_blend_group(fyx_ctx *ctx, uint32_t n, const uint32_t *anims, const float *weights, uint32_t *out_group);
int32_t fyx_anim_set_blend_weights(fyx_ctx *ctx, uint32_t group, uint32_t n, const float *weights);
/* AnimationContainer::update_animations(dt) for every animation of the context.  The touched nodes are marked
 * changed exactly like fyx_set_local_trs; follow with fyx_update_transforms / fyx_render_prep. */
int32_t fyx_animate(fyx_ctx *ctx, float dt);

/* ---- N3: draw-prep after the cull (SURVEY §8f) ------------------------------------------------ */
/* What RenderDataBundleStorage::push and RenderDataBundle::write_uniforms do per visible surface on the CPU
 * (renderer/bundle.rs:1248-1278, 483-487), for nodes with ONE surface: the instances of a frustum's visible
 * list grouped by bundle, each with its sort index, world matrix and view_projection * world. */

/* Meshes with several surfaces (Mesh::surfaces): Mesh::collect_render_data pushes ONE SurfaceInstanceData per surface, each
 * into the bundle of ITS (material, surface data, render path) key and with ITS bones, all with the node's sort index; the
 * world matrix is the identity for a skinned surface and the node's global transform otherwise (scene/mesh/mod.rs:726-805).
 * For node idx[i] the surfaces are entries [first[i], first[i+1]) of bundle_ids / skin_surface (first has count + 1 entries):
 * bundle_ids[k] = the dense bundle id of surface k, skin_surface[k] = the fyx surface id (fyx_add_skinned_surface) whose
 * palette skins it, FYX_NONE (or skin_surface == NULL) = unskinned.  Nodes never listed keep the default: one surface in the
 * node's bundle id (fyx_set_bundle_ids), skinned iff the node has a skinned surface.  A count of 0 surfaces restores the default.
 * fyx_set_topology keeps a node's surfaces with its node index while the node is alive before and after the call; any other
 * node index starts again from the default. */
int32_t fyx_set_node_surfaces(fyx_ctx *ctx, uint32_t count, const uint32_t *idx, const uint32_t *first, const uint32_t *bundle_ids,
                              const uint32_t *skin_surface);
/* Per-node bundle id = the host's dense id for the (material, surface data, render path) key that push()
 * hashes (renderer/bundle.rs:1253-1257); every node starts in bundle 0.  idx NULL = nodes 0..count-1. */
int32_t fyx_set_bundle_ids(fyx_ctx *ctx, uint32_t count, const uint32_t *idx, const uint32_t *bundle_ids);
/* Ask the culls that follow to also record where each visible node lives in HBM (4 more bytes written per
 * visible entry); required before fyx_pack_instances. */
int32_t fyx_enable_instances(fyx_ctx *ctx, uint32_t enable);

typedef struct fyx_bundle {
    uint32_t id;          /* the bundle id given to fyx_set_bundle_ids */
    uint32_t first;       /* first instance of the bundle in the packed arrays */
    uint32_t count;       /* RenderDataBundle::instances.len() */
    uint32_t reserved;
    uint64_t sort_index;  /* RenderDataBundle::sort_index: that of the instance pushed first (bundle.rs:1264-1268), i.e.
                           * first in the DFS order given to fyx_set_dfs_order, else the lowest node index */
} fyx_bundle;

typedef struct fyx_instances {
    uint32_t count;             /* instances: one per (visible node, surface) */
    uint32_t n_bundles;         /* non-empty bundles */
    const uint32_t *node;       /* [count]   SurfaceInstanceData::node_handle (index) */
    const uint64_t *sort_index; /* [count]   RenderContext::calculate_sorting_index(global_position) (bundle.rs:118-127) */
    const float *matrices;      /* [count*32] per instance: world_transform (identity for a skinned surface,
                                 * scene/mesh/mod.rs:733-737), then view_projection * world_transform (bundle.rs:485);
                                 * both column-major — the first 128 bytes of the instance uniform block */
    const fyx_bundle *bundles;  /* [n_bundles] ascending id; bundle b owns instances [first, first+count) in unspecified order */
} fyx_instances;

/* Pack the visible list of `frustum` (of the most recent cull, made with instances enabled) for an observer
 * with the given view and view-projection matrices (ObserverPosition, renderer/observer.rs). */
int32_t fyx_pack_instances(fyx_ctx *ctx, uint32_t frustum, const float *view_m16, const float *view_projection_m16);
/* [count] ordinal of each packed instance's surface within its node (host copy; 0 everywhere without fyx_set_node_surfaces). */
int32_t fyx_get_instance_surfaces(fyx_ctx *ctx, uint32_t frustum, const uint32_t **out_ordinal);
/* Result of the last fyx_pack_instances for that frustum: pointers to pinned host copies ... */
int32_t fyx_get_instances(fyx_ctx *ctx, uint32_t frustum, fyx_instances *out);
/* ... or to the device-resident arrays (count / n_bundles still come back as host values). */
int32_t fyx_get_instances_device(fyx_ctx *ctx, uint32_t frustum, fyx_instances *out);

/* Bone matrices of the packed instances, as RenderDataBundle::write_uniforms lays them out (renderer/bundle.rs:484-496):
 * every instance whose node has a skinned surface gets a block of FYX_MAX_BONES (255 = ShaderDefinition::
 * MAX_BONE_MATRICES) column-major mat4 — its SurfaceInstanceData::bone_matrices, then all-zero matrices — and an
 * unskinned instance gets none (bone_matrices_block = None).  Uses the palettes of the last fyx_build_palettes /
 * fyx_render_prep; call after fyx_pack_instances.  The surface that skins an instance is the one named by
 * fyx_set_node_surfaces, else the node's first skinned surface. */
typedef struct fyx_bone_blocks {
    uint32_t count;                    /* instances == fyx_instances.count */
    uint32_t n_blocks;                 /* skinned instances */
    const uint32_t *block_of_instance; /* [count] block of packed instance i, FYX_NONE = unskinned          (device memory) */
    const float *blocks;               /* [n_blocks * 255 * 16], 16 320 bytes per block, in unspecified order (device memory) */
} fyx_bone_blocks;
int32_t fyx_pack_bone_matrices(fyx_ctx *ctx, uint32_t frustum);
int32_t fyx_get_bone_matrix_blocks_device(fyx_ctx *ctx, uint32_t frustum, fyx_bone_blocks *out);
/* Host copy of one instance's block (out_255x16 may be NULL to ask only whether it has one). */
int32_t fyx_get_bone_matrix_block(fyx_ctx *ctx, uint32_t frustum, uint32_t instance, float *out_255x16, uint32_t *out_has_block);

/* The same packing for every shadow map of the last fyx_cull_shadow_casters, in one call (the reference builds a whole
 * RenderDataBundleStorage::from_graph per map, renderer/shadow/spot.rs:142-159, shadow/point.rs:173-197).  Map m is packed
 * exactly as fyx_pack_instances packs a frustum for an observer whose view_matrix is the map's look_at_rh (spot or cube
 * face) and whose view_projection is maps[m].view_projection: one instance per (listed node, surface), grouped by bundle id,
 * bundle sort index by the fyx_set_dfs_order rule.  The shadow cull must have been made with fyx_enable_instances (it then
 * records each entry's slot, 4 bytes per entry).  The instances of all maps live in one packed array: the fyx_instances of
 * map m points at its part, and bundles[k].first counts from the map's first instance.  Synchronous; a fixed number of
 * launches per group of consecutive maps whose (map, bundle id) bins stay under 2^25 (one group unless the id space is huge).
 * FYX_ERR_STATE when there is no shadow cull, it was made without fyx_enable_instances, fyx_set_topology has run since it
 * (its slots are stale) or a frame is still in flight. */
int32_t fyx_pack_shadow_instances(fyx_ctx *ctx);
/* Result of the last fyx_pack_shadow_instances for map `map` (FYX_ERR_INVALID_ARGUMENT when map >= the map count): pinned host
 * copies of the map's part, valid until the next host getter call on the same pack, or the next pack ... */
int32_t fyx_get_shadow_instances(fyx_ctx *ctx, uint32_t map, fyx_instances *out);
/* ... or pointers into the device arrays. */
int32_t fyx_get_shadow_instances_device(fyx_ctx *ctx, uint32_t map, fyx_instances *out);
/* [count] ordinal of each of the map's instances' surface within its node (host copy, valid until the next host getter call on
 * the same pack, or the next pack). */
int32_t fyx_get_shadow_instance_surfaces(fyx_ctx *ctx, uint32_t map, const uint32_t **out_ordinal);
/* Bone matrices of the shadow instances.  Unlike write_uniforms, which copies a surface's palette into every instance that
 * uses it (16 320 bytes per instance), there is ONE block per fyx surface (fyx_add_skinned_surface): block s is surface s's
 * palette of the last fyx_build_palettes / fyx_render_prep followed by zero matrices, bit for bit the block write_uniforms
 * builds (renderer/bundle.rs:484-496).  In the fyx_bone_blocks of a map, block_of_instance[i] is the id of the surface that
 * skins instance i (FYX_NONE = unskinned) and n_blocks is the number of surfaces.  FYX_ERR_STATE before
 * fyx_pack_shadow_instances (and, for the getters, before this call). */
int32_t fyx_pack_shadow_bone_matrices(fyx_ctx *ctx);
int32_t fyx_get_shadow_bone_matrix_blocks_device(fyx_ctx *ctx, uint32_t map, fyx_bone_blocks *out);
int32_t fyx_get_shadow_bone_matrix_block(fyx_ctx *ctx, uint32_t map, uint32_t instance, float *out_255x16, uint32_t *out_has_block);

/* The same for every observer of the last fyx_cull_scene_observers (made with fyx_enable_instances), in one call: observer o
 * is packed exactly as fyx_pack_instances packs a frustum for (view[o], view_projection[o]).  The getters and the bone
 * blocks (one per fyx surface) work as those of the shadow maps, with the observer in place of the map.  FYX_ERR_STATE when
 * there is no observer cull, it was made without fyx_enable_instances, fyx_set_topology has run since it or a frame is
 * still in flight. */
int32_t fyx_pack_scene_observer_instances(fyx_ctx *ctx);
int32_t fyx_get_scene_observer_instances(fyx_ctx *ctx, uint32_t observer, fyx_instances *out);
int32_t fyx_get_scene_observer_instances_device(fyx_ctx *ctx, uint32_t observer, fyx_instances *out);
int32_t fyx_get_scene_observer_instance_surfaces(fyx_ctx *ctx, uint32_t observer, const uint32_t **out_ordinal);
int32_t fyx_pack_scene_observer_bone_matrices(fyx_ctx *ctx);
int32_t fyx_get_scene_observer_bone_matrix_blocks_device(fyx_ctx *ctx, uint32_t observer, fyx_bone_blocks *out);
int32_t fyx_get_scene_observer_bone_matrix_block(fyx_ctx *ctx, uint32_t observer, uint32_t instance, float *out_255x16,
                                                 uint32_t *out_has_block);

/* ---- Dynamic batching (BatchingMode::Dynamic) ----------------------------------------------------------------------
 * Mesh::collect_render_data batches a surface instead of pushing it when the mesh is BatchingMode::Dynamic, has no blend
 * shapes, the surface has no bones and it has fewer than 256 vertices (scene/mesh/mod.rs:739-753).  In every pass (camera,
 * each shadow map, each observer) it then copies the surface's vertices with transform_vertex (scene/mesh/mod.rs:109-126:
 * position by world.transform_point, normal and tangent xyz by world.transform_vector, tangent w kept) and appends them, with
 * the surface's triangles shifted by the vertex count so far, to one shared surface per vertex layout (DynamicSurfaceCache,
 * renderer/cache/mod.rs:225-281) in the bundle keyed by (material, sort index, render path); consecutive push_triangles into
 * the same bundle extend the last instance instead of adding one (renderer/bundle.rs:1177-1243; scene/mesh/mod.rs:804-833).
 *
 * A registered surface is uploaded once and stays in device memory.  The instance packs (fyx_pack_instances,
 * fyx_pack_shadow_instances, fyx_pack_scene_observer_instances) then no longer pack it as an instance (the other instances keep
 * their surface ordinals) and build each segment's dynamic batches instead, as one from_graph would. */
typedef struct fyx_dynamic_layout { /* the VertexBuffer layout, as transform_vertex sees it */
    uint32_t stride;
    /* cast_attribute (scene/mesh/buffer.rs:1338-1357) checks only an attribute's size in bytes, never its declared type: give
     * an offset whenever the attribute's size is 12 bytes (position, normal) or 16 bytes (tangent), else FYX_NONE */
    uint32_t position_offset; /* 12 bytes: transform_point */
    uint32_t normal_offset;   /* 12 bytes: transform_vector */
    uint32_t tangent_offset;  /* 16 bytes: xyz transform_vector, w kept */
} fyx_dynamic_layout;
/* Register surface `surface_ordinal` (the Mesh::surfaces index) of `node` as batched.  batch_key = the host's dense id
 * (< 2^24) for the (material, render path) pair; layout_id = the host's dense id (< 2^16) for the layout's hash, which selects
 * the shared surface.  verts = n_verts records of layout->stride bytes; triangles = 3 u32 per triangle.  FYX_ERR_INVALID_ARGUMENT
 * for n_verts >= 256 (the reference pushes such a surface), a surface that fyx_set_node_surfaces names as skinned, an ordinal
 * the node does not have, a (node, ordinal) already registered, a layout_id given before with another layout, and a
 * batch_key given before with another layout_id (the reference's push_vertex_raw would panic, scene/mesh/buffer.rs:506-517),
 * and triangles that would not end below 2^32 u32 words of the context's triangle pool (dropped registrations keep their words
 * until the next pack reuses the space).
 * Registrations stay with their node index across fyx_set_topology; a node it removes drops them.  A surface that a later
 * fyx_set_node_surfaces removes or names skinned is pushed again (its registration is kept but not used).  The call copies the
 * data before it returns.  out_id may be NULL. */
int32_t fyx_add_dynamic_surface(fyx_ctx *ctx, uint32_t node, uint32_t surface_ordinal, uint32_t batch_key, uint32_t layout_id,
                                const fyx_dynamic_layout *layout, uint32_t n_verts, const void *verts, uint32_t n_triangles,
                                const uint32_t *triangles, uint32_t *out_id);
/* Drop the registrations of the listed nodes (nodes NULL = of every node).  A batch key or layout id that no registration uses
 * any more may come back with another layout id or layout.  The pools' space is reused once dropped surfaces are the larger part. */
int32_t fyx_clear_dynamic_surfaces(fyx_ctx *ctx, uint32_t count, const uint32_t *nodes);

typedef struct fyx_dynamic_bundle {
    uint32_t batch_key, layout_id;
    uint32_t first, count; /* the bundle's instances, counted from the segment's first */
    uint64_t sort_index;   /* that of the node pushed first into the bundle */
} fyx_dynamic_bundle;
typedef struct fyx_dynamic_instance {
    uint32_t node;            /* the first node of the run of pushes the instance covers */
    uint32_t triangle_offset; /* ElementRange::Specific in its layout's triangle stream */
    uint32_t triangle_count;
    uint32_t reserved;
} fyx_dynamic_instance;
typedef struct fyx_dynamic_stream { /* one layout's shared surface of the segment */
    uint32_t layout_id, stride, n_vertices, n_triangles;
    const void *vertices;       /* [n_vertices * stride] bytes */
    const uint32_t *triangles;  /* [n_triangles * 3] */
} fyx_dynamic_stream;
/* One segment's (frustum, map or observer) dynamic batches.  Bundles in the order of their first push; streams in ascending
 * layout_id, one per layout the segment uses.  Offsets and indices count from the segment's first vertex and first triangle of
 * that layout: that is the reference's shared surface when the pass is the first of the frame to use the layout; otherwise
 * the reference's numbers are these plus the earlier passes' vertex and triangle counts of the layout. */
typedef struct fyx_dynamic_batches {
    uint32_t n_bundles, n_instances, n_streams, reserved;
    const fyx_dynamic_bundle *bundles;
    const fyx_dynamic_instance *instances;
    const fyx_dynamic_stream *streams; /* host memory (its vertices / triangles point where the getter says) */
} fyx_dynamic_batches;
/* The dynamic batches of the last fyx_pack_instances of `frustum`, fyx_pack_shadow_instances (map) or
 * fyx_pack_scene_observer_instances (observer): pinned host copies valid until the next host getter call on the same pack or
 * the next pack, or (_device) pointers into device memory.  The streams array of a host getter's result stays valid until the
 * next host getter call on that pack, that of a device getter's until the next device getter call.  Refusals are the instance
 * getters'. */
int32_t fyx_get_dynamic_batches(fyx_ctx *ctx, uint32_t frustum, fyx_dynamic_batches *out);
int32_t fyx_get_dynamic_batches_device(fyx_ctx *ctx, uint32_t frustum, fyx_dynamic_batches *out);
int32_t fyx_get_shadow_dynamic_batches(fyx_ctx *ctx, uint32_t map, fyx_dynamic_batches *out);
int32_t fyx_get_shadow_dynamic_batches_device(fyx_ctx *ctx, uint32_t map, fyx_dynamic_batches *out);
int32_t fyx_get_scene_observer_dynamic_batches(fyx_ctx *ctx, uint32_t observer, fyx_dynamic_batches *out);
int32_t fyx_get_scene_observer_dynamic_batches_device(fyx_ctx *ctx, uint32_t observer, fyx_dynamic_batches *out);

/* ---- Sprites and 2D rectangles: the other push_triangles callers ------------------------------------------------------
 * Sprite::collect_render_data (scene/sprite.rs:322-405) and dim2::Rectangle::collect_render_data (scene/dim2/rectangle.rs:
 * 323-410) push one quad per node, after should_be_rendered, through the same push_triangles as Dynamic meshes: four vertices,
 * triangles [0,1,2] [0,2,3], render path Forward, sort index calculate_sorting_index(global_position).  A quad node is one more
 * item of its pass's dynamic batches: it shares bundle_map and last_bundle_id with the Dynamic surfaces of the pass, and its
 * layout's stream with any Dynamic surface given the same layout_id.  The getters above return the quads; a quad node is
 * never an ordinary instance (fyx_instances) of any pack, and surfaces fyx_set_node_surfaces later gives it are not packed.
 *   Gates: a sprite pushes nothing in a shadow pass, nor, in any pass, when its FYX_NODE_CAST_SHADOWS is off (sprite.rs:
 *   327-329); a rectangle pushes nothing in a shadow pass (rectangle.rs:328-330).  Shadow passes (renderer/mod.rs:128-131):
 *   every map of fyx_pack_shadow_instances, and a fyx_pack_instances frustum culled with FYX_PASS_SHADOW; never an observer.
 *   Culling: both are tested with AABB::unit() transformed by the global transform (sprite.rs:314-316 through base.rs:741-750;
 *   rectangle.rs:310-317), never with the sprite's size: the host keeps each quad node's unit box.
 *   Vertices (lx = uv_rect[0], rx = uv_rect[0] + uv_rect[2], ty = uv_rect[1], by = uv_rect[1] + uv_rect[3], f32 adds), in the
 *   corner order (+,+) (-,+) (-,-) (+,-):
 *     SpriteVertex, 40 bytes: position f32x3 = the global position (the translation column, unchanged) in every vertex,
 *       tex_coord f32x2, params f32x4 = (size, rotation, +-0.5, +-0.5), color u8x4.  tex_coord x: flip_x ? lx : rx,
 *       flip_x ? rx : lx, flip_x ? rx : lx, flip_x ? lx : rx.
 *     RectangleVertex, 24 bytes: position f32x3 = global_transform.transform_point((+-0.5, +-0.5, 0)), tex_coord f32x2, color
 *       u8x4.  tex_coord x is the sprite's mirrored: flip_x ? rx : lx, flip_x ? lx : rx, flip_x ? lx : rx, flip_x ? rx : lx.
 *     tex_coord y of both: flip_y ? by : ty for vertices 0 and 1, flip_y ? ty : by for vertices 2 and 3.
 *   The layout of a kind, in fyx_dynamic_layout terms: {40, 0, FYX_NONE, FYX_NONE} for sprites, {24, 0, FYX_NONE, FYX_NONE}
 *   for rectangles.  Layout ids and batch keys are shared with fyx_add_dynamic_surface: an id or key is free again only when
 *   neither a registration nor a quad node uses it. */
#define FYX_SPRITE_3D        1u /* scene::sprite::Sprite */
#define FYX_SPRITE_RECTANGLE 2u /* scene::dim2::rectangle::Rectangle */
typedef struct fyx_sprite {
    uint32_t kind;        /* FYX_SPRITE_3D | FYX_SPRITE_RECTANGLE */
    uint32_t batch_key;   /* < 2^24, the host's id for (material, Forward) */
    uint32_t layout_id;   /* < 2^16, the host's id for the kind's vertex layout */
    uint32_t flip;        /* bit 0 flip_x, bit 1 flip_y */
    float uv_rect[4];     /* position.x, position.y, size.x, size.y */
    float size, rotation; /* sprite only */
    uint8_t color[4];     /* r, g, b, a */
    uint32_t reserved;
} fyx_sprite;             /* 48 bytes */
/* Make nodes idx[0..count) (idx NULL = nodes 0..count-1) quad nodes with records[k], or update their records.  A change of
 * uv_rect, color, size, rotation or flip only rewrites the records; a new quad node, or a change of kind, batch_key or
 * layout_id, rebuilds the push-order tables at the next pack.  FYX_ERR_INVALID_ARGUMENT, with nothing changed, for: an
 * unknown kind; a node out of range, not alive or listed twice; a node with fyx_add_dynamic_surface registrations, with
 * surfaces from fyx_set_node_surfaces or with a skinned surface; a batch_key >= 2^24 or layout_id >= 2^16; a layout_id in use
 * with another layout; a batch_key in use with another layout_id.  Records stay with their node index across
 * fyx_set_topology; a node it removes drops its record.  fyx_add_dynamic_surface refuses a quad node. */
int32_t fyx_set_sprites(fyx_ctx *ctx, uint32_t count, const uint32_t *idx, const fyx_sprite *records);
/* Make the listed nodes (nodes NULL = every node) ordinary nodes again. */
int32_t fyx_clear_sprites(fyx_ctx *ctx, uint32_t count, const uint32_t *nodes);

/* ---- multi-GPU: one context per GPU, one process per GPU ------------------------------------- */
/* The node array is sharded (sub-trees + replicated ancestors, SURVEY §8e); each context culls its
 * shard; the per-frustum visible lists are all-gathered with NCCL over NVLink so every rank holds
 * the whole list.  Rank 0 obtains an id, the host broadcasts it, every rank calls fyx_comm_init. */
#define FYX_COMM_ID_BYTES 128
int32_t fyx_comm_get_unique_id(void *out_id128);
/* Collective.  The exchange buffers are built at the first gathered frame that follows (also collective: every rank
 * issues gathered frames in lockstep) and sized for every rank's node count at that time; call fyx_comm_init again on
 * every rank after a topology change that grows a shard. */
int32_t fyx_comm_init(fyx_ctx *ctx, int32_t nranks, int32_t rank, const void *id128);
/* How this context exchanges the lists (bit set), decided collectively at the first gathered frame:
 *   FYX_COMM_NCCL          NCCL is initialised (always; it is also the bootstrap channel of the other two)
 *   FYX_COMM_PEER_STORES   the device-side all-gather is done by direct stores into the peers' cudaIpc-mapped list
 *                          buffers over NVLink (no host synchronisation, no padded slots); otherwise ncclAllGather
 *   FYX_COMM_HOST_SEGMENT  the host copy of the gathered lists is assembled in one node-wide host segment: every rank
 *                          DMA-copies its own lists there over its own PCIe link
 *   FYX_COMM_UNDECIDED     no gathered frame has run yet
 * Environment (read by fyx_comm_init): FYX_EXCHANGE=nccl keeps the collective on NCCL, FYX_HOSTSEG=0 keeps private
 * host copies. */
#define FYX_COMM_NCCL 1u
#define FYX_COMM_PEER_STORES 2u
#define FYX_COMM_HOST_SEGMENT 4u
#define FYX_COMM_UNDECIDED 8u
uint32_t fyx_comm_mode(const fyx_ctx *ctx);
/* The most recent COMPLETED exchange of this rank, timed with CUDA events on the collective stream (waits for it). */
typedef struct fyx_comm_stats {
    uint64_t epoch;          /* number of the gathered frame */
    uint64_t entries_own;    /* visible entries this rank contributed (all frusta) */
    uint64_t entries_total;  /* entries of the gathered lists (all frusta) */
    uint64_t egress_bytes;   /* bytes this rank stored into OTHER ranks' memory: 4 * entries_own * (nranks - 1) (peer form) */
    float device_ms;         /* from the first kernel / collective of the exchange to its last one, incl. waiting for peers */
    uint32_t mode;           /* fyx_comm_mode at that time */
} fyx_comm_stats;
int32_t fyx_comm_get_stats(fyx_ctx *ctx, fyx_comm_stats *out);
/* All-gather the visible lists of the last cull.  Collective: every rank calls it for the same frame. */
int32_t fyx_allgather_visible(fyx_ctx *ctx);
/* Gathered list of frustum f: concatenation over ranks (device-resident and, if readback, on the host). */
int32_t fyx_get_visible_gathered(fyx_ctx *ctx, uint32_t frustum, const uint32_t **out_idx, uint32_t *out_count);
int32_t fyx_get_visible_gathered_device(fyx_ctx *ctx, uint32_t frustum, const uint32_t **d_idx, uint32_t *out_count);

#ifdef __cplusplus
}
#endif
#endif /* FYROX_B200_H */
