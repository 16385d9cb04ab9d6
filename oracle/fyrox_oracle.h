/*
 * fyrox_oracle.h — CPU restatement of Fyrox's render-prep hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing in the product (fyrox_b200/, include/) may
 * include, link or call this.  Only tests/, __graft_entry__.smoke() and the
 * cpu_baseline / --impl reference legs of bench.py use it, and only as the
 * checker / reported CPU baseline.
 *
 * Parity status: the reference (Rust, nalgebra 0.35 — semver range, no lock
 * file, sources absent from /root/reference) cannot be compiled here (no
 * cargo/rustc).  This restatement follows the reference source line by line
 * (each function cites file:line under /root/reference) and is PINNED against
 * the reference's own unit-test vectors K1..K15 (SURVEY.md §8c, see
 * tests/test_oracle_kat.py; K11-K15 pin the animation step's curves / wrapf / quaternion product,
 * fyrox_anim_oracle.c).  The functions the reference does not test
 * (calculate_local_transform, bone palette, LBS, Mesh world AABB,
 * should_be_rendered, from_graph, light collection, instance data,
 * Animation::tick, track fetch, pose blending and application) are
 * "parity unpinned": they follow source only.  nalgebra's accumulation orders (Appendix A of SURVEY.md) are the
 * restatement's definition.
 *
 * All matrices are 16 floats, column-major (nalgebra storage): M[r,c] = m[c*4+r].
 * Build: gcc -O2 -ffp-contract=off (Rust/LLVM never contracts mul+add to FMA).
 */
#ifndef FYROX_ORACLE_H
#define FYROX_ORACLE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ORC_NONE 0xFFFFFFFFu

typedef struct { float n[3]; float d; } orc_plane;                 /* fyrox-math/src/plane.rs:24-27 */
typedef struct { orc_plane planes[6]; float corners[8][3]; } orc_frustum; /* frustum.rs:26-30 */
typedef struct { float min[3]; float max[3]; } orc_aabb;           /* aabb.rs:26-29 */

/* Transform's TRS + pivots (fyrox-impl/src/scene/transform.rs:79-127). Quaternions are (i,j,k,w). */
typedef struct {
    float local_position[3];
    float local_rotation[4];
    float local_scale[3];
    float pre_rotation[4];
    float post_rotation_matrix[9]; /* column-major 3x3, the cached inverse post-rotation matrix (transform.rs:160-172) */
    float rotation_offset[3];
    float rotation_pivot[3];
    float scaling_offset[3];
    float scaling_pivot[3];
} orc_transform;

/* Vertex attribute offsets inside an interleaved vertex (scene/mesh/vertex.rs:140-210). */
typedef struct {
    uint32_t stride;
    uint32_t position_offset;     /* f32 x3 */
    uint32_t normal_offset;       /* f32 x3 */
    uint32_t bone_weights_offset; /* f32 x4 */
    uint32_t bone_indices_offset; /* u8  x4 */
} orc_vertex_layout;

/* ---- plane.rs ---- */
int   orc_plane_from_abcd(float a, float b, float c, float d, orc_plane *out);
float orc_plane_dot(const orc_plane *p, const float pt[3]);
void  orc_plane_intersection_point(const orc_plane *a, const orc_plane *b, const orc_plane *c, float out[3]);

/* ---- frustum.rs ---- */
int  orc_frustum_from_view_projection_matrix(const float m[16], orc_frustum *out);
void orc_frustum_default(orc_frustum *out);
int  orc_frustum_is_intersects_point_cloud(const orc_frustum *f, const float *pts_xyz, size_t n);
int  orc_frustum_is_intersects_aabb(const orc_frustum *f, const orc_aabb *aabb);
int  orc_frustum_is_intersects_aabb_offset(const orc_frustum *f, const orc_aabb *aabb, const float off[3]);
int  orc_frustum_is_contains_point(const orc_frustum *f, const float pt[3]);

/* ---- aabb.rs ---- */
void orc_aabb_default(orc_aabb *a);
void orc_aabb_unit(orc_aabb *a);
void orc_aabb_add_point(orc_aabb *a, const float p[3]);
void orc_aabb_add_box(orc_aabb *a, const orc_aabb *b);
void orc_aabb_corners(const orc_aabb *a, float out[8][3]);
int  orc_aabb_is_valid(const orc_aabb *a);
int  orc_aabb_is_degenerate(const orc_aabb *a);
int  orc_aabb_is_contains_point(const orc_aabb *a, const float p[3]);
void orc_aabb_transform(const orc_aabb *a, const float m[16], orc_aabb *out);

/* ---- nalgebra pieces on the path (Appendix A) ---- */
void orc_mat4_identity(float out[16]);
void orc_mat4_mul(const float a[16], const float b[16], float out[16]);
void orc_mat4_transform_point(const float m[16], const float p[3], float out[3]);
void orc_quat_to_rotation_matrix(const float q[4], float r9[9]);
void orc_look_at_rh(const float eye[3], const float target[3], const float up[3], float out[16]);
void orc_perspective(float aspect, float fovy, float znear, float zfar, float out[16]);
void orc_orthographic(float l, float r, float b, float t, float zn, float zf, float out[16]);

/* ---- scene/transform.rs ---- */
void orc_transform_identity(orc_transform *t);
void orc_transform_calculate_local(const orc_transform *t, float out[16]);

/* ---- renderer/bundle.rs:118-127 ---- */
uint64_t orc_calculate_sorting_index(const float view[16], const float global_position[3]);

/* ---- scene graph (pointer tree of heap nodes, as the reference) ---- */
typedef struct orc_graph orc_graph;

enum { ORC_KIND_PIVOT = 0, ORC_KIND_MESH = 1 };

orc_graph *orc_graph_new(void);                 /* root pivot = index 0 (graph/mod.rs:408-424) */
void       orc_graph_free(orc_graph *g);
uint32_t   orc_graph_capacity(const orc_graph *g);
uint32_t   orc_graph_root(const orc_graph *g);
uint32_t   orc_graph_add_node(orc_graph *g, int kind);                 /* graph/mod.rs:2044-2088 */
void       orc_graph_link_nodes(orc_graph *g, uint32_t child, uint32_t parent); /* :2114-2131 */
void       orc_graph_remove_node(orc_graph *g, uint32_t node);         /* :2091-2111 (frees subtree) */
/* Bulk construction: nodes 1..capacity-1 are created in index order and linked in index order
 * (children lists ordered by index); node 0 is the root.  parent[i]==ORC_NONE leaves i an orphan
 * (only legal for i==0 in a well-formed graph). kind bit: flags bit5 (see FLAG_ below). */
orc_graph *orc_graph_build(uint32_t capacity, const uint32_t *parent, const uint32_t *flags,
                           const uint32_t *render_mask, const float *local_m16, const float *local_aabb6);

/* node flag bits shared with the C-ABI (include/fyrox_b200.h) */
#define ORC_FLAG_VISIBILITY      (1u << 0)
#define ORC_FLAG_ENABLED         (1u << 1)
#define ORC_FLAG_FRUSTUM_CULLING (1u << 2)
#define ORC_FLAG_CAST_SHADOWS    (1u << 3)
#define ORC_FLAG_ALIVE           (1u << 4)
#define ORC_FLAG_RENDERABLE      (1u << 5)   /* node kind emits render data (Mesh) */
#define ORC_FLAG_LIGHT           (1u << 6)   /* node is a BaseLight (point / spot / directional) */
#define ORC_FLAG_REFLECTION_PROBE (1u << 15) /* node is a ReflectionProbe (renderer/bundle.rs:918-925) */
#define ORC_FLAG_STATIC_BATCH    (1u << 7)   /* Mesh::batching_mode == BatchingMode::Static (scene/mesh/mod.rs:701-725) */

/* property setters; the three tracked ones push messages like TrackedProperty::deref_mut (base.rs:343-352) */
void orc_node_set_local_matrix(orc_graph *g, uint32_t n, const float m16[16]);
void orc_node_set_local_transform(orc_graph *g, uint32_t n, const orc_transform *t);
void orc_node_set_visibility(orc_graph *g, uint32_t n, int v);
void orc_node_set_enabled(orc_graph *g, uint32_t n, int v);
void orc_node_set_frustum_culling(orc_graph *g, uint32_t n, int v);
void orc_node_set_cast_shadows(orc_graph *g, uint32_t n, int v);
void orc_node_set_render_mask(orc_graph *g, uint32_t n, uint32_t mask);
void orc_node_set_inv_bind_pose(orc_graph *g, uint32_t n, const float m16[16]);
void orc_mesh_set_local_aabb(orc_graph *g, uint32_t mesh, const orc_aabb *a);   /* stands for Mesh::local_bounding_box cache */
/* adds a surface; verts may be NULL (no vertex data); returns surface index */
uint32_t orc_mesh_add_surface(orc_graph *g, uint32_t mesh, uint32_t n_bones, const uint32_t *bones,
                              uint32_t n_verts, const void *verts, const orc_vertex_layout *layout);
/* recompute Mesh::local_bounding_box from all surface vertex positions (mesh/mod.rs:631-656) */
void orc_mesh_recalc_local_aabb(orc_graph *g, uint32_t mesh);

/* update */
void orc_graph_update(orc_graph *g);                     /* Graph::update → process_node_messages (graph/mod.rs:1303-1399) */
void orc_graph_update_hierarchical_data(orc_graph *g);   /* :1272-1292, from root */
void orc_graph_drop_messages(orc_graph *g);

/* queries */
void     orc_node_global_transform(const orc_graph *g, uint32_t n, float out[16]);
void     orc_node_local_matrix(const orc_graph *g, uint32_t n, float out[16]);
int      orc_node_global_visibility(const orc_graph *g, uint32_t n);
int      orc_node_is_globally_enabled(const orc_graph *g, uint32_t n);
void     orc_node_world_bounding_box(const orc_graph *g, uint32_t n, orc_aabb *out);
uint32_t orc_node_parent(const orc_graph *g, uint32_t n);
int      orc_node_should_be_rendered(const orc_graph *g, uint32_t n, const orc_frustum *f, uint32_t render_mask);
void     orc_graph_global_scale(const orc_graph *g, uint32_t n, const float *local_scales_xyz, float out[3]);

/* RenderDataBundleStorage::from_graph reduced to its visible-node emission (bundle.rs:873-1009):
 * DFS pre-order from the root; Mesh nodes that pass should_be_rendered (+ cast_shadows on shadow
 * passes, mesh/mod.rs:691-698) are appended.  Returns the number of visible nodes (may exceed cap;
 * only the first cap are written). */
size_t orc_from_graph(const orc_graph *g, const orc_frustum *f, uint32_t render_mask, int shadow_pass,
                      uint32_t *out_idx, size_t cap);

/* bone palette (mesh/mod.rs:781-793) and CPU LBS (mesh/mod.rs:501-522 for positions; normals follow
 * standard.shader:192-195 in the same op order) */
uint32_t orc_mesh_bone_matrices(const orc_graph *g, uint32_t mesh, uint32_t surface, float *out_m16);
uint32_t orc_mesh_skin(const orc_graph *g, uint32_t mesh, uint32_t surface, float *out_pos3, float *out_nrm3);
void     orc_node_set_lod_group(orc_graph *g, uint32_t node, uint32_t n_levels, const float *begin, const float *end,
                                const uint32_t *obj_begin, const uint32_t *objects);          /* scene/base.rs:805-807 */
void     orc_lod_filter(const orc_graph *g, const float observer_translation[3], float z_near, float z_far, uint8_t *filter);
size_t   orc_from_graph_lod(const orc_graph *g, const orc_frustum *f, uint32_t render_mask, int shadow_pass,
                            const float observer_translation[3], float z_near, float z_far, uint32_t *out_idx, size_t cap); /* N4: bundle.rs:898-916,988-1004 */
/* N4: the reflection-probe selection of from_graph (renderer/bundle.rs:918-925): ORC_NONE = no probe contains the observer */
uint32_t orc_select_reflection_probe(const orc_graph *g, const float observer_translation[3]);
size_t   orc_collect_lights(const orc_graph *g, const orc_frustum *f, uint32_t *out_idx, size_t cap);   /* N4: renderer/bundle.rs:926-974 */
uint64_t orc_node_instance(const orc_graph *g, uint32_t node, const float view[16], const float vp[16],
                           float world[16], float wvp[16]);   /* N3: mesh/mod.rs:700,731-737 + bundle.rs:483-487 */
void     orc_mesh_accurate_world_bounding_box(const orc_graph *g, uint32_t mesh, orc_aabb *out);

/* free-standing skin of one vertex array with a given palette (used by the bench CPU baseline) */
void orc_skin_vertices(const float *palette_m16, uint32_t n_verts, const void *verts,
                       const orc_vertex_layout *layout, float *out_pos3, float *out_nrm3);
/* N3: one instance per surface (scene/mesh/mod.rs:726-805) and its bone block */
uint64_t orc_node_surface_instance(const orc_graph *g, uint32_t node, uint32_t surface, const float view[16], const float vp[16],
                                   float world[16], float wvp[16], int *out_skinned);
int orc_surface_bone_block(const orc_graph *g, uint32_t mesh, uint32_t surface, float out[255 * 16]);
/* N3: the zero-padded 255-mat4 block of one instance (renderer/bundle.rs:484-496); 0 = the node has no skinned surface */
int orc_instance_bone_block(const orc_graph *g, uint32_t mesh, float out[255 * 16]);
/* N4: blend-shape stage of the standard shader (standard.shader:167-173), then orc_skin_vertices; weights already / 100 */
void orc_skin_vertices_blend(const float *pal, uint32_t n_verts, const void *verts, const orc_vertex_layout *l, uint32_t n_shapes,
                             const uint16_t *records, uint32_t layer_stride, const float *weights, float *out_pos, float *out_nrm);

/* ---- N2: animation sampling (fyrox_anim_oracle.c) ---- */
enum { ORC_KEY_CONSTANT = 0, ORC_KEY_LINEAR = 1, ORC_KEY_CUBIC = 2 };            /* CurveKeyKind, fyrox-math/src/curve.rs:33-45 */
typedef struct { float location, value; uint32_t kind; float left_tangent, right_tangent; } orc_curve_key; /* curve.rs:57-63 */
enum { ORC_TV_REAL = 0, ORC_TV_VECTOR2, ORC_TV_VECTOR3, ORC_TV_VECTOR4, ORC_TV_QUAT_EULER, ORC_TV_QUAT }; /* TrackValueKind, container.rs:41-54 */
enum { ORC_BIND_POSITION = 0, ORC_BIND_SCALE = 1, ORC_BIND_ROTATION = 2 };      /* ValueBinding, value.rs:358-374 */
typedef struct {
    uint32_t target_node;  /* TrackBinding::target */
    uint32_t binding;      /* ORC_BIND_* */
    uint32_t value_kind;   /* ORC_TV_* */
    uint32_t enabled;      /* TrackBinding::enabled */
    uint32_t n_curves;     /* TrackDataContainer::curves.len() */
    uint32_t first_key[4]; /* curve c = keys[first_key[c] .. first_key[c] + n_keys[c]) sorted by location */
    uint32_t n_keys[4];
} orc_track;
typedef struct orc_animation orc_animation;

float orc_wrapf(float n, float min_limit, float max_limit);                       /* fyrox-math/src/lib.rs:179-203 */
float orc_lerpf(float a, float b, float t);                                       /* lib.rs:206-208 */
float orc_cubicf(float p0, float p1, float t, float m0, float m1);                /* lib.rs:212-221 */
float orc_key_interpolate(const orc_curve_key *l, const orc_curve_key *r, float t); /* curve.rs:87-136 */
float orc_curve_value_at(const orc_curve_key *keys, uint32_t n, float location, uint32_t *hint); /* curve.rs:252-309 */
void  orc_quat_from_euler_xyz(const float euler[3], float q[4]);                  /* lib.rs:725-740 */
void  orc_track_value_blend(int is_quat, float a[4], const float b[4], float w);  /* value.rs:201-227,449-454 */
int   orc_track_fetch(const orc_track *t, const orc_curve_key *keys, float time, uint32_t hints[4], float out[4]); /* container.rs:162-301 */
orc_animation *orc_animation_new(const orc_track *tracks, uint32_t n_tracks, const orc_curve_key *keys, uint32_t n_keys);
void  orc_animation_free(orc_animation *a);
void  orc_animation_set_time_position(orc_animation *a, float time);              /* fyrox-animation/src/lib.rs:432-440 */
void  orc_animation_set_time_slice(orc_animation *a, float start, float end);     /* lib.rs:445-452 */
void  orc_animation_set_speed(orc_animation *a, float s);
void  orc_animation_set_looped(orc_animation *a, int l);
void  orc_animation_set_enabled(orc_animation *a, int e);
void  orc_animation_set_track_enabled(orc_animation *a, uint32_t track, int e);
float orc_animation_time_position(const orc_animation *a);
int   orc_animation_is_enabled(const orc_animation *a);
void  orc_update_animations(orc_animation **anims, uint32_t n, float dt, orc_graph *g, orc_transform *transforms,
                            uint32_t n_nodes);                                    /* scene/animation/mod.rs:83-88,107-179 */
void  orc_blend_group_update(orc_animation **anims, const float *weights, uint32_t n, float dt, orc_graph *g,
                             orc_transform *transforms, uint32_t n_nodes);       /* machine/mod.rs:344-382, node/blend.rs:136-166, pose.rs:41-101 */
/* The same passes inside one frame: frame_dirty = Transform::dirty per node, shared by every pass of the frame (the
 * player and the machines) and cleared by the caller when the graph updates; NULL = a frame with this pass alone,
 * which is what the two calls above are. */
void  orc_update_animations_in_frame(orc_animation **anims, uint32_t n, float dt, orc_graph *g, orc_transform *transforms,
                                     uint32_t n_nodes, uint8_t *frame_dirty);
void  orc_blend_group_update_in_frame(orc_animation **anims, const float *weights, uint32_t n, float dt, orc_graph *g,
                                      orc_transform *transforms, uint32_t n_nodes, uint8_t *frame_dirty);
int   orc_node_is_alive(const orc_graph *g, uint32_t n);

/* ---- "soa-omp-NT": the same arithmetic on flat arrays with OpenMP (fyrox_oracle_mt.c) — a best-effort multi-core CPU
 * baseline, NOT how the reference runs (it is single-threaded); results equal the restatement above bit for bit ---- */
typedef struct orc_mt orc_mt;
orc_mt  *orc_mt_new(uint32_t n, uint32_t root, const uint32_t *parent, const uint32_t *flags, const uint32_t *mask,
                    const float *local_m16, const float *local_aabb6);
void     orc_mt_free(orc_mt *m);
void     orc_mt_set_threads(orc_mt *m, int threads);
void     orc_mt_set_local_matrices(orc_mt *m, uint32_t count, const uint32_t *idx, const float *m16);
void     orc_mt_set_inv_bind(orc_mt *m, uint32_t node, const float m16[16]);
uint32_t orc_mt_add_surface(orc_mt *m, uint32_t mesh, uint32_t n_bones, const uint32_t *bones, uint32_t n_verts,
                            const void *verts, const orc_vertex_layout *layout);
void     orc_mt_update(orc_mt *m);
size_t   orc_mt_cull(const orc_mt *m, const orc_frustum *f, uint32_t render_mask, int shadow_pass, uint32_t *out, size_t cap);
void     orc_mt_skin_surface(const orc_mt *m, uint32_t surface, float *out_pos3, float *out_nrm3);
void     orc_mt_skin_all(const orc_mt *m);
void     orc_mt_get(const orc_mt *m, uint32_t node, float g16[16], orc_aabb *world_aabb, uint32_t *gflags /* vis | en<<1 | reach<<2 */);

#ifdef __cplusplus
}
#endif
#endif
