// fyx_internal.h — device data layout and kernel launchers shared by fyx_api.cu / fyx_kernels.cu.
//
// HBM layout (DESIGN.md §3).  Nodes live in SLOT order = sorted by (depth, node index), so every
// hierarchy level is one contiguous, coalesced range and a parent is always in an earlier range.
// All per-node columns are SoA planes indexed by slot:
//   L[3], G[3]   float4 rows of the affine local / global matrix (48 B each; bottom row implicit)
//   la[3], wa[3] float2 (min_i,max_i) pairs of the local / world AABB (24 B each)
//   parent       u32 parent slot (FYX_NONE = none)      flags  u32 (input bits + computed bits)
//   mask         u32 Base::render_mask                  gidx   u32 node index emitted to visible lists
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "../../include/fyrox_b200.h"
#include "fyx_math.cuh"
#include "fyx_anim_plan.hpp"
#include "fyx_dyn_plan.hpp"
#include "fyx_skin_plan.hpp"
#include "fyx_slots.hpp"

namespace fyx {

// internal flag bits (above the public ones)
constexpr uint32_t F_DIRTY_SELF = 1u << 11; // local matrix / topology changed since the last update
constexpr uint32_t F_DIRTY = 1u << 12;      // in a changed sub-tree during the last update
constexpr uint32_t F_SKINNED = 1u << 13;    // Mesh with at least one skinned surface
constexpr uint32_t F_ROOT = 1u << 14;       // Graph::root

constexpr int kCountStride = 32; // u32s between per-frustum counters (128 B: one L2 line each)
constexpr int kBlock = 256;

// ------------------------------------------------------------------------------------------------
// Programmatic dependent launch: the kernels of a frame form a chain of true data dependencies (level l
// needs level l-1, the fold needs every level, the palettes the bones, the skinning the palettes), several
// of them tiny.  Each is launched with programmatic stream serialization: it lets the next kernel's CTAs be
// scheduled right away (pdl_trigger) and waits for the previous kernel's results only where it first needs
// them (pdl_wait) — launch latency and the loads that do not depend on the predecessor overlap its tail.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

template <class... Params, class... Args>
static void launch_pdl(void (*kernel)(Params...), unsigned grid, unsigned block, size_t smem, cudaStream_t s, Args... args)
{
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(block);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    cudaLaunchKernelEx(&cfg, kernel, static_cast<Params>(args)...);
}

struct NodeArrays {
    uint32_t cap; // number of slots (alive nodes)
    uint32_t *parent;
    uint32_t *flags;
    uint32_t *mask;
    uint32_t *gidx;
    float4 *L[3];
    float4 *G[3];
    float2 *la[3];
    float2 *wa[3];
};

struct CullParams {
    int nf;
    FrustumDev f[FYX_MAX_FRUSTA];
    uint32_t *out[FYX_MAX_FRUSTA]; // visible lists
    uint32_t *out_slot[FYX_MAX_FRUSTA]; // the same entries as HBM slots (nullptr unless fyx_enable_instances)
    uint32_t *counts;              // counts[f * kCountStride]
    float one, negzero;            // 1.0f, -0.0f: run-time operands of the unfusable packed FMAs (fyx_math.cuh)
};

struct SkinArrays {
    // bone table (one entry per (surface, bone))
    uint32_t n_entries;
    const uint32_t *bone_slot; // slot of the bone node, FYX_NONE ⇒ identity
    const float4 *ib[3];       // inverse bind pose rows
    float *palette;            // n_entries * 16 f32, column-major mat4 (the reference's bone_matrices layout)
    // input vertices: blocks of 128 vertices (32 four-vertex groups), 11 rows of 32 float4 (512 B) each:
    //   rows 0-2 position x,y,z   rows 3-5 normal x,y,z   rows 6-9 weight 0..3   row 10 the 4x u8 bone indices;
    // element l of a row belongs to group l of the block and holds the value of its 4 vertices.  A warp reads
    // a row with one perfectly coalesced 512 B access and every 32 B sector exactly once (44 B/vertex).
    // A block may instead hold the exact code of fyx_vcode.cuh (5 136 B at the same stride; SkinTile::vcoded).
    const float4 *vblk;
    float *opos, *onrm;        // skinned streams, packed xyz (each surface padded to a multiple of 4 vertices)
    // N4 blend shapes (optional): f16 position / normal offsets per (shape, vertex) in blocks of 128 vertices x 6 rows
    // (px,py,pz,nx,ny,nz) x 32 groups x 4 halfs = 1536 B per (shape, block); weights = BlendShape::weight / 100
    const uint2 *bs;
    const float *bs_w;
};

constexpr uint32_t kBsBlockU2 = 6 * 32; // uint2 per (shape, block)
void launch_bs_layout(cudaStream_t s, uint32_t n_verts, uint32_t n_shapes, uint32_t layer_stride, const uint16_t *d_records, uint2 *d_dst, uint32_t bs_blocks);

struct FoldArrays {
    uint32_t n; // skinned mesh nodes
    const uint32_t *node_slot;
    const uint32_t *bone_begin; // n+1 offsets into bone_slot
    const uint32_t *bone_slot;  // bones of all skinned surfaces of the node, in surface order
    // bones the reference's DFS visits AFTER their mesh contribute the position they had before this update
    // (scene/mesh/mod.rs:676-682 reads the stored value): per entry an index into stale_pos, FYX_NONE = use the new one
    const uint32_t *stale_idx;  // nullptr when no such bone exists
    const float4 *stale_pos;
};

// N2 animation sampling (fyx_anim.cu; AnimTrackDev / AnimStateDev in fyx_anim_plan.hpp); launch_animate returns its launches
struct AnimArrays {
    uint32_t n_tracks, n_anims, n_nodes;
    const fyx_curve_key *keys;
    AnimTrackDev *tracks;
    AnimStateDev *state;
    uint4 *hints;                    // TrackBinding::fetch_hints per track
    float4 *values;                  // sampled value per track
    uint32_t *value_ok;              // fetch returned Some
    const uint32_t *track_bind_kind; // binding | value_kind << 8
    // animated nodes (distinct live targets) and, per node, its tracks in (animation, track) order
    const uint32_t *node_slot;
    const uint32_t *node_begin;
    const uint32_t *node_tracks;
};
uint32_t launch_animate(cudaStream_t s, const NodeArrays &a, const AnimArrays &an, fyx_trs *trs_by_slot,
                        const fyx_transform_statics *st_by_slot, float dt, uint32_t *d_err);

// N3 draw-prep (fyx_drawprep.cu): one frustum's visible list -> instances grouped by bundle
struct InstParams {
    uint32_t n;                     // visible entries
    const uint32_t *vis_node;       // the visible list (node indices)
    const uint32_t *vis_slot;       // the same entries as slots
    const uint32_t *bundle_of_slot; // nullptr = every node in bundle 0
    const uint32_t *rank_of_slot;   // pre-order DFS rank (fyx_set_dfs_order); nullptr = node index order
    // surfaces of a node (Mesh::surfaces): ms_range[slot] = (first, count) into ms_bundle / ms_skin; count 0 (or ms_range == nullptr)
    // = ONE surface in the node's bundle id, skinned iff the node has a skinned surface (surf_of_slot)
    const uint2 *ms_range;
    const uint32_t *ms_bundle, *ms_skin;
    const uint32_t *surf_of_slot;   // the node's first skinned fyx surface, FYX_NONE = none
    float view[16], vp[16];         // column-major
    uint32_t n_bundle_ids;
    // scratch (hist and first_key are cleared by the caller: 0 / ~0)
    uint32_t *hist;                 // n_bundle_ids: instances per bundle, then the scatter cursor
    unsigned long long *first_key;  // n_bundle_ids: min (rank << 32 | list position) of the bundle
    uint32_t *offset;               // n_bundle_ids: first instance of the bundle
    uint64_t *tmp_sort;             // n
    // outputs
    uint32_t *o_node;
    uint64_t *o_sort;
    uint32_t *o_surf;               // ordinal of the instance's surface within its node
    uint32_t *o_skin;               // fyx surface id whose palette skins the instance, FYX_NONE = unskinned
    float4 *o_mats;                 // 8 float4 per instance: world (4 columns), view_projection * world (4 columns)
    fyx_bundle *o_bundles;
    uint32_t *o_totals;             // [2] bundles and instances (of the group)
    // ---- segments (fyx_pack_shadow_instances): the list is the entries of shadow maps [map0, map0 + n_seg), each map one
    // segment with its own observer; bin = segment * n_bundle_ids + bundle.  vis_node / vis_slot / tmp_sort start at the
    // group's first entry, `n` counts the group's entries.
    const fyx_shadow_map *maps;     // all maps of the shadow cull (first / count, view_projection)
    const float *views;             // [maps * 16] the maps' view matrices
    uint32_t map0, n_seg;
    uint32_t base_inst, base_bundle; // instances and bundles of the groups packed before this one
    uint32_t *seg_inst;             // [n_seg] instances per segment (keys pass, cleared by the caller)
    uint32_t *seg_first;            // [n_seg] first instance of the segment (all groups)
    uint32_t *seg_bfirst;           // [n_seg] first bundle of the segment (all groups)
    uint2 *tile_sum;                // [tiles] (instances, bundles) per tile of kScanTile bins, then their exclusive prefix
    // ---- Dynamic batching (fyx_add_dynamic_surface): surfaces batched by the pack's dynamic pass are not instances.
    // dyn_of_slot nullptr = none registered; else the node's dense dynamic index (FYX_NONE = none), whose registered
    // surface ordinals are dyn_ordinal[dyn_item_first[d] .. dyn_item_first[d + 1]); ordinal FYX_NONE = every surface (a quad node)
    const uint32_t *dyn_of_slot, *dyn_item_first, *dyn_ordinal;
};

// One pack's dynamic pass over its segments (DynItemDev / DynLayoutDev in fyx_dyn_plan.hpp): mark (the segments' dynamic nodes
// and counts), then, once the host has placed every segment's items, hash tables and (segment, layout) streams, order + bundles
// (one CTA per segment) and geometry.
struct DynParams {
    // registrations
    const uint32_t *dyn_of_slot, *item_first; // [slots], [D + 1]
    const DynItemDev *items;
    const DynLayoutDev *layouts;
    uint32_t n_layouts, words; // words: bitmap u32 per segment (ceil(D / 32))
    const unsigned char *vtx;
    const uint32_t *tri;
    const fyx_sprite *quads;   // [slots] the quad nodes' records (fyx_set_sprites)
    uint32_t shadow;           // the pack's segments are shadow passes; one flag serves them all because every caller of
                               // pack_segments packs passes of one kind (see there)
    // the pack's list, cut into segments
    uint32_t n, n_seg;
    const uint32_t *vis_slot;
    const uint32_t *seg_first; // [n_seg + 1] first list entry of each segment, then the list's end
    const float *views;        // [n_seg * 16] each segment's view matrix
    uint32_t *bitmap;          // [n_seg * words]
    uint32_t *counts;          // [n_seg * n_layouts * 3]: items, vertices, triangles
    // placed by the host from counts
    const uint32_t *seg_item0;   // [n_seg + 1] first item (all segments' items one after the other)
    const uint32_t *seg_hash0;   // [n_seg] first entry of the segment's two hash tables
    const uint32_t *seg_hmask;   // [n_seg] entries per table - 1 (a power of two)
    const uint64_t *stream_vtx;  // [n_seg * n_layouts] first output byte of each (segment, layout) vertex stream
    const uint32_t *stream_tri;  // [n_seg * n_layouts] first output triangle of each (segment, layout) stream
    // per item (in push order, at seg_item0 + position), cleared by the host where noted
    uint32_t *ord_item, *voff, *toff, *bord, *run_of, *run_item, *run_bundle, *run_tend;
    uint32_t *bcur;              // per bundle: instances, then the first instance / cursor (cleared to 0)
    uint64_t *sidx, *key2;
    unsigned long long *hkey;    // cleared to ~0
    uint32_t *hval;              // cleared to ~0
    // outputs
    fyx_dynamic_bundle *o_bundles;   // at seg_item0[seg]
    fyx_dynamic_instance *o_inst;    // at seg_item0[seg]
    uint32_t *o_seg;                 // [n_seg * 2] bundles, instances
    unsigned char *o_vtx;
    uint32_t *o_tri;
};
void launch_dyn_mark(cudaStream_t s, const NodeArrays &a, const DynParams &dp);
// order, then geometry when `meshes` (the tables hold registered surfaces) and the quad kernel when `quads`; returns the launches
int launch_dyn_batches(cudaStream_t s, const NodeArrays &a, const DynParams &dp, uint32_t n_items, bool meshes, bool quads);
// keys + scan (o_totals), then the scatter.  One segment: the one-CTA scan; segmented (the shadow maps of one group): the
// device-wide scan of the bins
constexpr uint32_t kScanTile = 4096; // bins per CTA of the device-wide scan
void launch_inst_count(cudaStream_t s, const NodeArrays &a, const InstParams &ip, bool segmented);
void launch_inst_scatter(cudaStream_t s, const NodeArrays &a, const InstParams &ip, bool segmented);
void launch_bone_block_index(cudaStream_t s, uint32_t n, const uint32_t *inst_skin, uint32_t *block_of_inst, uint32_t *counter);
// one CTA per block; inst_skin / block_of_inst nullptr = block i is surface i's
void launch_bone_blocks(cudaStream_t s, uint32_t n, const uint32_t *inst_skin, const uint2 *surf_bones, const float *palette, const uint32_t *block_of_inst,
                        float *blocks);

// Sub-forest plan (plan_subforest, fyx_slots.hpp): the deep levels of the hierarchy — small sub-trees such as skeletons — are
// cut into groups of whole sub-trees; one CTA walks all levels of its group with CTA-wide barriers instead of one kernel
// launch per level.
struct SubforestPlan {
    uint32_t n_ctas = 0, n_levels = 0, first_level = 0; // deep levels = [first_level, first_level + n_levels)
    const uint2 *rng = nullptr;                        // [cta][level] = slot range (begin, end)
};
void launch_update_subforest(cudaStream_t s, const NodeArrays &a, const SubforestPlan &sf, bool update_all, const CullParams *cull);

// ---- launchers (fyx_kernels.cu) ----
void launch_update_level(cudaStream_t s, const NodeArrays &a, uint32_t lo, uint32_t hi, bool update_all,
                         const CullParams *cull /* nullptr = no fused cull */);
// the observers of fyx_set_observers, one per frustum, by value
struct Observers {
    uint32_t n;
    fyx_observer o[FYX_MAX_FRUSTA];
};
void launch_select_probes(cudaStream_t s, const NodeArrays &a, const Observers &obs, uint32_t *best /* [n], cleared to 0 by the caller: node index + 1 */);
void launch_cull_lights(cudaStream_t s, const NodeArrays &a, const CullParams &cp, uint32_t *const *d_out_ptrs, uint32_t *counts);

// N4 shadow casters (fyx_cull_shadow_casters): one record per light node, in pool order
struct ShadowLightDev {
    uint32_t slot;
    uint32_t kind; // FYX_LIGHT_*
    float m22;     // 1 / tan(fovy / 2), evaluated on the host
    float distance_or_radius;
    fyx_csm_options csm; // directional lights: the cascades' FrustumSplitOptions
};
// one camera or reflection probe of fyx_cull_scene_observers, in the order of the observers they give
struct ObserverRecDev {
    uint32_t slot;
    uint32_t kind;              // FYX_OBSERVER_*
    uint32_t mode;              // camera: FYX_PROJECTION_*; probe: FYX_PROBE_UPDATE_*
    uint32_t enabled;           // camera: Camera::is_enabled
    uint32_t rendered;          // probe: emitted since its record was set or its update forced
    uint32_t emitted;           // probe: emitted by the current call (k_observer_views); folded into `rendered` once it succeeds
    float m22_or_vertical_size; // camera: 1 / tan(fov / 2) (evaluated on the host) or vertical_size
    float z_near, z_far;
    float v[3];                 // camera: frame size (0,0 = the call's); probe: rendering_position
};
// the camera of the cascaded shadow maps (fyx_cull_shadow_casters_csm); enabled = 0: directional lights get no maps
struct CsmCameraDev {
    uint32_t enabled;
    uint32_t projection;        // FYX_PROJECTION_*
    float m22_or_vertical_size; // perspective: 1 / tan(fov / 2), evaluated on the host; orthographic: vertical_size
    float z_near, z_far;
    float frame_size[2];
    float view[16];
    fyx_frustum fallback; // Frustum::default() as planes + corners: a cascade slice's unwrap_or_default (shadow/csm.rs:215-219)
};
// A many-map cull (the shadow maps of one camera, the scene's observers, the observers' shadow maps): a one-CTA table kernel
// writes up to `max maps` map rows with their frusta; the count pass reads every node once and counts its entries per map;
// the scan places the lists; the emit pass re-tests the warps that had an entry and writes them.  MapParams is what the node
// passes, the scan and the pruner table read, and what the table kernels write.
struct MapParams {
    // the map table
    fyx_frustum *scratch; // [max maps] the map frusta as planes + corners
    FrustumDev *frusta;   // [max maps] each with the render mask of what renders the map
    fyx_shadow_map *maps; // [max maps]
    float *views;         // [max maps * 16] the maps' view matrices, for the instance pack
    uint32_t *n_maps;     // one u32
    // node passes: per-map counts (each on its own 128 B line), then the lists
    uint32_t *counts;     // [max maps * kCountStride]
    uint32_t *warp_any;   // [warps]: the warp's nodes are in at least one map (written by the count pass, read by the emit pass)
    uint32_t *total;      // one u32: entries of all maps
    uint32_t *entries;    // [total], sized by the host from the count pass
    uint32_t *entry_slot; // [total] the same entries as HBM slots; nullptr unless fyx_enable_instances
    uint32_t cam_mask;    // kFormShadow: the one camera's render mask, tested once per node (the other forms: frusta[m].cam_mask)
    // ---- per-map LOD filter and static-batch pruning (unused by the unpruned kernels).
    // A pruner is a LOD object or an FYX_NODE_STATIC_BATCH node; pruners have dense ids in slot order.
    struct Prune {
        const uint32_t *col;    // per slot: the nearest pruner on the node's path (id | kPrSelf when the node is that pruner), FYX_NONE = none
        const uint32_t *slot;   // per pruner: its slot
        const uint32_t *anc;    // per pruner: the nearest strict pruner ancestor, FYX_NONE = none
        const float2 *range;    // per slot: LOD range (begin NaN = none); nullptr = no node has one
        uint32_t *rows;         // [pruner][2][words]: maps hiding the pruner itself, then maps hiding its children
        uint32_t words;         // u32 words per row (ceil(max maps / 32))
        float *obs;             // [max maps * 5]: the map's observer for the LOD filter (translation, z_near, z_far)
        uint32_t *err;          // the context's error word (E_SHADOW_LIST)
    } pr;
};
// What only the table kernels of the shadow culls read (k_shadow_frusta, k_scene_shadow_maps): the light table and the
// shadow loop's settings; for one camera also that camera and its cascades
struct ShadowParams {
    const ShadowLightDev *lights;
    uint32_t n_lights;
    FrustumDev cam;      // fyx_cull_shadow_casters*: the camera frustum of the last cull (planes + cam_mask)
    FrustumDev fallback; // Frustum::default(): from_view_projection_matrix(..).unwrap_or_default() (renderer/bundle.rs:893-896)
    float cam_t[3];      // fyx_cull_shadow_casters*: the camera's translation
    float spot_distance, point_distance;
    uint32_t spot_enabled, point_enabled;
    const fyx_trs *trs; // the node's last TRS record per slot; nullptr = none sent (identity scale)
    CsmCameraDev csm;   // fyx_cull_shadow_casters*: the cascades' camera; the scene form takes its `fallback` for every observer's
};
// The scene's observers (fyx_cull_scene_observers): a many-map cull with one map per observer, in kFormObservers (each
// observer's own mask, no cast_shadows).  What only the observer kernels read:
struct ObserverParams {
    ObserverRecDev *recs;       // [n_recs] due probes' and cameras' records: probes in pool order, then cameras
    uint32_t n_recs;
    float frame_size[2];        // the call's frame size
    float probe_m22;            // 1 / tan(FRAC_PI_2 / 2), evaluated on the host
    fyx_frustum fallback;       // Frustum::default(): from_view_projection_matrix(..).unwrap_or_default()
    fyx_scene_observer *table;  // [max observers]
    uint32_t *light_counts;     // [max observers * kCountStride]: light-list counts, then write cursors
    uint32_t *best;             // [max observers]: environment map node + 1 (0 = none)
    uint32_t *light_total;      // one u32
    uint32_t *light_raw;        // [light_total] the light lists in emission order
    uint32_t *light_entries;    // [light_total] the same, each list in ascending node index
};
// The shadow maps of the scene's observers (fyx_cull_scene_shadow_casters): a many-map cull in kFormSceneShadow (each map's
// frustum carries the render mask of its observers).  Beside ShadowParams, what only its table kernel reads and writes:
struct SceneShadowCand {   // one (observer, light-list entry)
    uint32_t observer;     // its row of the observer table
    uint32_t light;        // its row of the light table, FYX_NONE = no record
    uint32_t n_maps, cascade;
    uint32_t hslot;        // spot or point with maps: its key's hash slot; else FYX_NONE
    uint32_t row;          // first map row, when it is the first of its key
};
struct SceneShadowParams {
    const fyx_scene_observer *table; // [n_obs] the observer table of the last fyx_cull_scene_observers
    uint32_t n_obs;
    const FrustumDev *frusta;        // [n_obs] the observers' frusta
    const uint32_t *light_entries;   // [n_cand] the observers' light lists, one after the other in table order
    uint32_t n_cand;
    const ObserverRecDev *recs;      // [n_recs] the records the table was built from
    uint32_t n_recs;
    float frame_size[2];             // the frame size of that call
    float probe_m22;
    uint32_t csm_enabled;
    CsmCameraDev *csm_cams;          // [n_obs] scratch: each observer's cascade camera
    SceneShadowCand *cand;           // [n_cand] scratch
    uint32_t *hash;                  // [hash_mask + 1] FYX_NONE-filled: the smallest candidate of each key
    uint32_t hash_mask;
    fyx_scene_shadow_map *refs;      // [6 n_cand] (observer, map) in render order
    uint32_t *n_refs;                // one u32
};
constexpr uint32_t kPrSelf = 1u << 31; // bit of MapParams::Prune::col: the node is the pruner itself
// The three forms of the node passes' one predicate:
//   kFormShadow (fyx_cull_shadow_casters*): every map carries the camera's mask, tested once per node;
//   kFormObservers (fyx_cull_scene_observers): the observers as maps, no shadow pass, each observer's own mask;
//   kFormSceneShadow (fyx_cull_scene_shadow_casters): the shadow pass, each map with its observer's own mask.
enum ShadowForm { kFormShadow, kFormObservers, kFormSceneShadow };
static_assert(kFormSceneShadow == 2, "tools/scene_shadow_bench.py finds that call's node passes by this value in their names (<.., 2>)");
// Every launcher returns the number of kernels it launched.
// The table kernels, one CTA each (pruned: the maps' LOD observers go to mp.pr.obs as well; the other two look at mp.pr.obs)
uint32_t launch_shadow_frusta(cudaStream_t s, const NodeArrays &a, const MapParams &mp, const ShadowParams &sp, bool pruned);
uint32_t launch_scene_shadow_maps(cudaStream_t s, const NodeArrays &a, const MapParams &mp, const ShadowParams &sp, const SceneShadowParams &ss);
uint32_t launch_observer_views(cudaStream_t s, const NodeArrays &a, const MapParams &mp, const ObserverParams &op);
// after the table kernel: the pruner table when pr_level_off is given (one launch per entry of pr_level_off that holds
// pruners, parents first), then the count pass; then the scan; then, once the host has sized the lists, the emit pass
uint32_t launch_map_count(cudaStream_t s, const NodeArrays &a, const MapParams &mp, ShadowForm form, const uint32_t *pr_level_off, uint32_t n_levels);
// The stand-alone camera cull over all slots: first, with pr_level_off, the camera's pruner table (pr.words = 1; pr.range
// nullptr = no LOD filter), one launch per entry of pr_level_off that holds pruners, parents first; then k_cull, which masks
// each node with its row (pr.col nullptr = no pruning)
uint32_t launch_cull(cudaStream_t s, const NodeArrays &a, const CullParams &cp, const MapParams::Prune &pr, const Observers &obs,
                     const uint32_t *pr_level_off, uint32_t n_levels);
uint32_t launch_map_scan(cudaStream_t s, const MapParams &mp);
uint32_t launch_map_emit(cudaStream_t s, const NodeArrays &a, const MapParams &mp, ShadowForm form, bool pruned);
// fyx_cull_scene_observers' own passes: the light counts and environment maps (emit = false) or the light lists (emit = true);
// the light scan; the light lists' sort (one CTA per observer)
uint32_t launch_observer_lights(cudaStream_t s, const NodeArrays &a, const MapParams &mp, const ObserverParams &op, bool emit);
uint32_t launch_observer_light_scan(cudaStream_t s, const MapParams &mp, const ObserverParams &op);
uint32_t launch_observer_light_sort(cudaStream_t s, const ObserverParams &op, uint32_t n_obs);
// after a call that succeeded: the probes it emitted count as rendered (probe.rs `updated`)
uint32_t launch_observers_commit(cudaStream_t s, ObserverRecDev *recs, uint32_t n_recs);
// the pruner column MapParams::Prune::col / anc from the pruners' slots: col must hold FYX_NONE everywhere; then one launch per
// hierarchy level [level_off[l], level_off[l + 1]) from level `first` on, parents first
void launch_pruner_mark(cudaStream_t s, uint32_t n_pruners, const uint32_t *pr_slot, uint32_t *col);
void launch_pruner_level(cudaStream_t s, const NodeArrays &a, uint32_t lo, uint32_t hi, uint32_t *col, uint32_t *anc);
void launch_fold_bones(cudaStream_t s, const NodeArrays &a, const FoldArrays &fa, const CullParams *cull);
void launch_snapshot_bones(cudaStream_t s, const NodeArrays &a, uint32_t n_late, const uint32_t *late_slot, float4 *stale_pos);
void launch_palette(cudaStream_t s, const NodeArrays &a, const SkinArrays &sk);
void launch_skin(cudaStream_t s, const SkinArrays &sk, const SkinTile *tiles, uint32_t n_tiles, uint32_t max_bones, bool blend_shapes);

void launch_scatter_locals(cudaStream_t s, const NodeArrays &a, uint32_t count, const uint32_t *d_idx,
                           const float *d_m16, const uint32_t *slot_of_node, uint32_t n_nodes, uint32_t *d_err);
void launch_scatter_trs(cudaStream_t s, const NodeArrays &a, uint32_t count, const uint32_t *d_idx, const void *d_payload /* fyx_trs or float4 quats */,
                        bool rot_only, fyx_trs *trs_by_slot /* device copy of the last records; may be nullptr unless rot_only */,
                        const fyx_transform_statics *statics_by_slot /* nullptr = defaults */, const uint32_t *slot_of_node,
                        uint32_t n_nodes, uint32_t *d_err);
// record e of d_val (`words` 32-bit words) into the slot of node d_idx[e] (d_idx nullptr = node e) of dst
void launch_scatter_words(cudaStream_t s, uint32_t *dst, uint32_t words, uint32_t count, const uint32_t *d_idx,
                          const uint32_t *d_val, const uint32_t *slot_of_node, uint32_t n_nodes);
// node flags: the public input bits except ALIVE are replaced, the computed bits kept
void launch_scatter_flags(cudaStream_t s, uint32_t *flags, uint32_t count, const uint32_t *d_idx,
                          const uint32_t *d_val, const uint32_t *slot_of_node, uint32_t n_nodes);
void launch_scatter_aabbs(cudaStream_t s, const NodeArrays &a, uint32_t count, const uint32_t *d_idx,
                          const float *d_aabb6, const uint32_t *slot_of_node, uint32_t n_nodes);
void launch_gather_globals(cudaStream_t s, const NodeArrays &a, uint32_t count, const uint32_t *d_idx,
                           const uint32_t *slot_of_node, uint32_t n_nodes, float *d_out_m16);
void launch_gather_aabbs(cudaStream_t s, const NodeArrays &a, uint32_t count, const uint32_t *d_idx,
                         const uint32_t *slot_of_node, uint32_t n_nodes, float *d_out6);
void launch_gather_flags(cudaStream_t s, const NodeArrays &a, uint32_t count, const uint32_t *d_idx,
                         const uint32_t *slot_of_node, uint32_t n_nodes, uint32_t *d_out);
// a surface's vertices into the raw blocks at first_vertex (a multiple of 4); with `code`, the blocks the load completes are
// then coded where they fit (fyx_vcode.cuh; vflag: one byte per block)
void launch_deinterleave(cudaStream_t s, uint32_t n_verts, const unsigned char *d_bytes, fyx_vertex_layout layout,
                         uint32_t n_bones, float4 *vblk, uint8_t *vflag, bool code, uint64_t first_vertex, uint32_t *d_err);
// every coded block back to raw (a context whose palettes need the register-load form of k_skin, which reads raw blocks)
void launch_vdecode_all(cudaStream_t s, float4 *vblk, uint8_t *vflag, uint64_t n_blocks);
void launch_tile_vcode(cudaStream_t s, SkinTile *tiles, uint32_t n_tiles, const uint8_t *vflag); // SkinTile::vcoded
constexpr uint32_t kSkinRingMaxBones = 64; // palettes up to this size: the prefetching form of k_skin, which reads coded blocks
constexpr int kVblkRows = 11;                    // float4 rows per block
constexpr int kVblkStride = kVblkRows * 32;      // float4 per block of 128 vertices
void launch_ib_rows(cudaStream_t s, uint32_t n, const float *d_m16, float4 *r0, float4 *r1, float4 *r2, uint32_t *d_err);
void launch_or_u32(cudaStream_t s, uint32_t *p, uint32_t bits);
// One record of at most 32 words, copied from a value of a plain type (fyx_trs, float2, ...)
struct WordRecord {
    uint32_t words;
    uint32_t w[32];
    template <class T> explicit WordRecord(const T &v) : words(sizeof(T) / 4), w{}
    {
        static_assert(sizeof(T) % 4 == 0 && sizeof(T) <= sizeof(w), "a record is a whole number of at most 32 words");
        memcpy(w, &v, sizeof(T));
    }
};
// dst[s] = (map && map[s] != FYX_NONE) ? src[map[s]] : def, records of def.words words: carries per-slot data over a topology
// change (slots move; fyx_set_topology), and with map == nullptr fills n records with def
void launch_permute_words(cudaStream_t s, void *dst, const void *src, const uint32_t *map, uint32_t n, const WordRecord &def);
void launch_compact_gathered(cudaStream_t s, const uint32_t *pad, uint32_t maxc, const uint32_t *counts_all, int nranks, int f,
                             uint32_t *dst);

// ---- multi-GPU exchange by peer stores (fyx_peer.cu) ----
constexpr int kPeerMaxRanks = 16;
struct PeerCtrl { // lives at the start of every rank's exchange allocation; written by the peers
    uint32_t counts[2][kPeerMaxRanks][FYX_MAX_FRUSTA]; // [epoch & 1][rank][frustum]
    uint32_t cnt_flag[2][kPeerMaxRanks];               // epoch of rank r's last count publication
    uint32_t done_flag[2][kPeerMaxRanks];              // epoch of rank r's last completed push into THIS rank's lists
    uint32_t totals[2][FYX_MAX_FRUSTA];                // gathered count per frustum (written by k_peer_wait)
};
constexpr size_t kPeerCtrlBytes = 4096;
static_assert(sizeof(PeerCtrl) <= kPeerCtrlBytes, "control block fits its page");
struct PeerParams {
    int nranks, rank, nf;
    uint32_t epoch;
    unsigned char *base[kPeerMaxRanks]; // every rank's exchange allocation as mapped into this process
    uint64_t total_cap;                 // entries per (slot, frustum) list: all ranks' slots together
    uint32_t nf_cap;
    const uint32_t *own_list[FYX_MAX_FRUSTA];
    const uint32_t *own_counts; // counts[f * kCountStride]
    uint32_t *cta_done;
    uint32_t *d_err;
};
__host__ __device__ inline PeerCtrl *peer_ctrl(const PeerParams &pp, int r) { return reinterpret_cast<PeerCtrl *>(pp.base[r]); }
__host__ __device__ inline uint32_t *peer_list(const PeerParams &pp, int r, uint32_t slot, uint32_t f)
{
    return reinterpret_cast<uint32_t *>(pp.base[r] + kPeerCtrlBytes) + ((size_t)slot * pp.nf_cap + f) * pp.total_cap;
}
void launch_peer_counts(cudaStream_t s, const PeerParams &pp);                   // publish this rank's counts, wait for everybody's
void launch_peer_push(cudaStream_t s, const PeerParams &pp, unsigned push_ctas); // store the lists into every rank's buffers, wait for everybody's

// error bits written by kernels into d_err
constexpr uint32_t E_NOT_AFFINE = 1u;
constexpr uint32_t E_BAD_BONE_INDEX = 2u;
constexpr uint32_t E_NONFINITE_VERTEX = 4u;
constexpr uint32_t E_PEER_TIMEOUT = 8u; // a rank never showed up in the peer exchange (bounded spin, fyx_peer.cu)
constexpr uint32_t E_SHADOW_LIST = 16u; // the pruned shadow emit pass found more entries for a map than its count pass (nothing written)

} // namespace fyx
