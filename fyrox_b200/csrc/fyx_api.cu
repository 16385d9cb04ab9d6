// fyx_api.cu — the C ABI of libfyrox_b200 (include/fyrox_b200.h): context, host-side bookkeeping
// (slot ordering by hierarchy depth, staging, surface tables) and stream-ordered kernel launches.
// No CPU fallback exists: every compute entry point launches the sm_90a kernels of fyx_kernels.cu.
#include <algorithm>
#include <array>
#include <limits>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <memory>
#include <new>
#include <set>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <utility>
#include <vector>

#include "fyx_frustum.cuh"
#include "fyx_hostseg.hpp"
#include "fyx_internal.h"

using namespace fyx;

// --------------------------------------------------------------------------------------------
// small utilities
// --------------------------------------------------------------------------------------------
namespace {

thread_local std::string g_create_error;

constexpr uint8_t kPrLod = 1, kPrBatch = 2; // fyx_ctx::pr_node

// Owners of the context's CUDA resources.  Each is move-only and frees what it holds when it dies; a move assignment swaps,
// so what the target held before dies with the moved-from source.  A failed allocation leaves the owner as it was.
struct DevBuf {
    void *p = nullptr;
    size_t bytes = 0;
    DevBuf() = default;
    DevBuf(DevBuf &&o) noexcept { *this = std::move(o); }
    DevBuf &operator=(DevBuf &&o) noexcept
    {
        std::swap(p, o.p);
        std::swap(bytes, o.bytes);
        return *this;
    }
    DevBuf(const DevBuf &) = delete;
    DevBuf &operator=(const DevBuf &) = delete;
    ~DevBuf()
    {
        if (p) cudaFree(p);
    }
    cudaError_t alloc(size_t n)
    {
        DevBuf fresh;
        const cudaError_t e = cudaMalloc(&fresh.p, n);
        if (e != cudaSuccess) {
            fresh.p = nullptr;
            return e;
        }
        fresh.bytes = n;
        *this = std::move(fresh);
        return cudaSuccess;
    }
    template <class T> T *as() const { return static_cast<T *>(p); }
};

// One per-node record per slot, for the data that fyx_set_topology carries to the nodes' new slots: local rows, TRS records,
// transform statics, bundle ids, LOD ranges.  `def` is the record of a node that was never given one.  A column that is not
// `live` has no records yet: its readers take the default (they are handed nullptr) and its first store fills it.
struct SlotColumn {
    DevBuf buf;
    WordRecord def;
    bool live = false;
    template <class T> explicit SlotColumn(const T &v) : def(v) {}
    int32_t ensure(fyx_ctx *c); // allocates c->n_slots records of def unless live
    int32_t carry(fyx_ctx *c, const uint32_t *old_of_new); // into the new slot order (c->n_slots), when live
    int32_t scatter(fyx_ctx *c, uint32_t count, const uint32_t *idx, const void *values); // the nodes' records, from the host
};

// The records kept with a value derived from them: the projection's one transcendental, evaluated on the host with the
// platform's tanf, and whether a probe is due
struct LightRec {
    fyx_light_source src;
    float m22; // 1 / tan(fovy / 2)
};
struct CameraRec {
    fyx_camera cam;
    float m22_or_vertical_size; // perspective: 1 / tan(fov / 2)
};
struct ProbeRec {
    fyx_reflection_probe probe;
    bool due; // set or forced since the observer table was built: its rendered bit starts at 0
};
constexpr fyx_csm_options kCsmDefault{0u, {5.0f, 25.0f, 64.0f}}; // FrustumSplitOptions::default() (scene/light/directional.rs:83-91)

// page-locked host memory
struct PinnedBuf {
    void *p = nullptr;
    size_t bytes = 0;
    PinnedBuf() = default;
    PinnedBuf(PinnedBuf &&o) noexcept { *this = std::move(o); }
    PinnedBuf &operator=(PinnedBuf &&o) noexcept
    {
        std::swap(p, o.p);
        std::swap(bytes, o.bytes);
        return *this;
    }
    PinnedBuf(const PinnedBuf &) = delete;
    PinnedBuf &operator=(const PinnedBuf &) = delete;
    ~PinnedBuf()
    {
        if (p) cudaFreeHost(p);
    }
    // at least n bytes; the contents are not kept.  The old buffer is freed first, so the caller must know that no copy
    // still uses it.  On failure the buffer is empty.
    cudaError_t ensure(size_t n)
    {
        if (n <= bytes) return cudaSuccess;
        *this = PinnedBuf{};
        const size_t nb = std::max<size_t>(4096, n + n / 2);
        const cudaError_t e = cudaHostAlloc(&p, nb, cudaHostAllocDefault);
        if (e != cudaSuccess) {
            p = nullptr;
            return e;
        }
        bytes = nb;
        return cudaSuccess;
    }
    template <class T> T *as() const { return static_cast<T *>(p); }
};

struct Event {
    cudaEvent_t h = nullptr;
    Event() = default;
    Event(Event &&o) noexcept { std::swap(h, o.h); }
    Event &operator=(Event &&o) noexcept
    {
        std::swap(h, o.h);
        return *this;
    }
    Event(const Event &) = delete;
    Event &operator=(const Event &) = delete;
    ~Event()
    {
        if (h) cudaEventDestroy(h);
    }
    cudaError_t create(unsigned flags)
    {
        Event fresh;
        const cudaError_t e = cudaEventCreateWithFlags(&fresh.h, flags);
        if (e == cudaSuccess) *this = std::move(fresh);
        else fresh.h = nullptr;
        return e;
    }
    operator cudaEvent_t() const { return h; }
};

struct Stream {
    cudaStream_t h = nullptr;
    Stream() = default;
    Stream(Stream &&o) noexcept { std::swap(h, o.h); }
    Stream &operator=(Stream &&o) noexcept
    {
        std::swap(h, o.h);
        return *this;
    }
    Stream(const Stream &) = delete;
    Stream &operator=(const Stream &) = delete;
    ~Stream()
    {
        if (h) cudaStreamDestroy(h);
    }
    cudaError_t create(int priority = 0)
    {
        Stream fresh;
        const cudaError_t e = priority ? cudaStreamCreateWithPriority(&fresh.h, cudaStreamNonBlocking, priority)
                                       : cudaStreamCreateWithFlags(&fresh.h, cudaStreamNonBlocking);
        if (e == cudaSuccess) *this = std::move(fresh);
        else fresh.h = nullptr;
        return e;
    }
    operator cudaStream_t() const { return h; }
};

enum { EV_START = 0, EV_UPLOAD, EV_UPDATE, EV_CULL, EV_PALETTE, EV_SKIN, EV_READBACK, EV_COUNT };

// Output of one cull: per-frustum visible lists + counters, device and (pinned) host side.  Two slots
// alternate so that the lists of frame i can travel to the host while frame i+1 is being culled.
struct VisSlot {
    DevBuf b_vis[FYX_MAX_FRUSTA];
    DevBuf b_vis_slot[FYX_MAX_FRUSTA]; // the same entries as HBM slots (fyx_enable_instances)
    bool have_slots = false;
    DevBuf d_counts;    // kCountStride * FYX_MAX_FRUSTA, each counter on its own 128 B line
    PinnedBuf h_counts; // FYX_MAX_FRUSTA
    PinnedBuf h_vis[FYX_MAX_FRUSTA];
    uint32_t nf = 0;
    bool counts_on_host = false, lists_on_host = false;
    // multi-GPU: the all-gathered lists of this frame (padded slots, packed list, host copy)
    DevBuf b_gath_pad[FYX_MAX_FRUSTA], b_gath[FYX_MAX_FRUSTA];
    uint32_t gath_count[FYX_MAX_FRUSTA] = {};
    PinnedBuf h_gath[FYX_MAX_FRUSTA];
    bool gathered = false, gathered_on_host = false;
    bool own_only = false; // FYX_FRAME_READBACK_OWN: the host copy of this frame is the rank's own lists
    Event ev_gather, ev_counts_all;
    uint64_t epoch = 0;            // number of this gathered frame (the same on every rank)
    bool via_peer = false;         // exchanged by peer stores (fyx_peer.cu), else NCCL
    uint32_t *gath_ptr[FYX_MAX_FRUSTA] = {}; // the gathered list on the device (peer allocation or b_gath)
    uint32_t counts_all[kPeerMaxRanks][FYX_MAX_FRUSTA] = {};
    bool counts_all_known = false;
    // host copy of the gathered lists through the node-wide segment (fyx_hostseg.hpp)
    bool host_copy_private = false; // the frame did not ask for a read-back: a later fetch copies the device list privately
    bool seg_published = false, seg_complete = false, own_in_seg = false;
    uint32_t *seg_own[FYX_MAX_FRUSTA] = {};
    bool pending = false; // written by a pipelined (async + read-back) frame that fyx_frame_wait has not collected yet
    uint64_t frame_no = 0;
    Event ev_cull, ev_counts, ev_done;
};

// N3: packed instances in segments, segment after segment (fyx_drawprep.inl): one segment for a camera frustum, one per
// map for the shadow maps
struct InstPack {
    DevBuf b_node, b_sort, b_mats, b_bundles, b_surf, b_skin;
    DevBuf b_block_of, b_blocks; // bone-matrix blocks of the instances
    std::vector<uint32_t> inst_first, bundle_first; // [segments + 1]
    const uint32_t *block_of = nullptr;             // [instances] block of each instance: b_block_of, or b_skin (one block per surface)
    uint32_t n_blocks = 0;
    // pinned host copies of one segment (node, sort, mats, bundles; surface ordinals) and the segment each holds
    PinnedBuf h[4], h_surf;
    uint32_t h_seg = FYX_NONE, h_surf_seg = FYX_NONE;
    bool valid = false, blocks_valid = false;
    uint32_t segments() const { return (uint32_t)inst_first.size() - 1; }
    // the dynamic batches of every segment (fyx_dynamic_batches): bundles and instances at dyn.item0[seg], each segment's
    // streams at dyn.stream0[seg] of dyn.streams with device pointers
    DevBuf b_dyn_bundles, b_dyn_inst, b_dyn_vtx, b_dyn_tri;
    DynPlacement dyn;
    std::vector<uint32_t> dyn_counts; // [segments * 2] bundles / instances
    PinnedBuf h_dyn[4];                     // bundles, instances, vertices, triangles of segment h_dyn_seg
    std::vector<fyx_dynamic_stream> dyn_out_host, dyn_out_dev; // the streams handed out by the last host / device getter
    uint32_t h_dyn_seg = FYX_NONE;
};

// N4: what a many-map cull leaves (fyx_drawprep.inl; MapParams in fyx_internal.h): the map table, the lists, their pinned
// copies and the maps' instance pack, a segment per map.  A call takes prepare, its own table kernel, the count pass and
// the scan (with what else it counts and scans), lists, the emit pass, commit.
struct MapCull {
    DevBuf b_scratch, b_frusta, b_maps, b_views, b_counts, b_warp_any;
    DevBuf b_small; // n, total, then words of the caller's (a third count it reads back with them)
    DevBuf b_entries, b_slots; // the lists as node indices and (with instances enabled) as HBM slots
    PinnedBuf h_small, h_maps, h_entries;
    uint32_t n = 0, total = 0; // maps, entries of all maps: set by lists, before the call has succeeded, so like every
                               // result here they may be read only behind `valid`
    bool valid = false, on_host = false, have_slots = false, slots_stale = false;
    InstPack pack;
    void invalidate() { valid = pack.valid = false; }
    void topology_changed() { slots_stale = true; } // the entries' slots are the old order's
    // buffers for up to max_maps maps, the node passes' parameters (the pruner table's too when pruned), counts cleared
    int32_t prepare(fyx_ctx *c, size_t max_maps, bool pruned, MapParams &mp);
    // waits for the scan, reads n, total (and the caller's words: n_small in all) and sizes the lists
    int32_t lists(fyx_ctx *c, MapParams &mp, uint32_t n_small);
    void commit(const fyx_ctx *c); // the call succeeded: the results are the context's
};

// Scratch of the instance packs, shared by all of them: per bin (histogram, first key, offset), per entry (sort index), per
// segment (instances, first instance, first bundle), the device-wide scan's tile sums, and the totals with a pinned copy
struct PackScratch {
    DevBuf hist, first_key, offset, tmp_sort, seg, tiles, totals;
    PinnedBuf h_totals;
    int32_t ensure(fyx_ctx *c, size_t bins, size_t entries, size_t segments);
    // the dynamic pass (DynParams): the host's small arrays, the bitmap and counts, the per-item scratch, the hash tables
    DevBuf dyn_small, dyn_bitmap, dyn_counts, dyn_items32, dyn_items64, dyn_hkey, dyn_hval;
    PinnedBuf h_dyn_counts;
};

// Dynamic batching (fyx_drawprep.inl): what push_triangles batches, the registrations of Dynamic meshes and the quad nodes
// (fyx_set_sprites) with the rules of fyx_dyn_plan.hpp, the quad nodes' full records by slot, which the quad kernel reads, the
// pools, and the device tables in push order (DynItemDev).  The tables are rebuilt by the first pack after invalidate(), which
// every input of the flush calls: the registrations, the quad nodes, the topology, the DFS order and the node surfaces.
struct DynBatches {
    DynRegistry reg;
    SlotColumn quads{fyx_sprite{}};
    DevBuf b_vtx, b_tri; // pools: vertex bytes, triangles (reg.vtx_used / reg.tri_used)
    bool stale = false;
    uint32_t n_nodes = 0, n_items = 0, n_quads = 0, n_layouts = 0; // of the device tables
    DevBuf b_of_slot, b_item_first, b_ordinal, b_items, b_layouts;

    void invalidate() { stale = true; }
    void topology_changed(const std::vector<uint32_t> &old_slot_of_node, const std::vector<uint32_t> &new_slot_of_node)
    {
        reg.topology_changed(old_slot_of_node, new_slot_of_node);
        invalidate();
    }
    int32_t compact(fyx_ctx *c);
    int32_t flush(fyx_ctx *c);
    int32_t pack(fyx_ctx *c, InstPack &o, const uint32_t *vis_slot, const float *views, const float *view, const std::vector<uint32_t> &first,
                 bool shadow);
};

// The skinned surfaces (fyx_add_skinned_surface) and what the frame kernels read of them: the vertex store, the bone tables,
// the blend-shape pools, and the tables plan_skin (fyx_skin_plan.hpp) derives from the surfaces and the topology, which
// commit rebuilds when `dirty`.  Surfaces and skinned_node stay with their node index across topology calls.
struct Skinning {
    std::vector<SkinSurface> surfaces;
    std::vector<uint8_t> skinned_node; // per node: has a skinned surface
    // vertex store: 128-vertex blocks with one flag byte each (raw or coded, fyx_vcode.cuh), the skinned output streams
    uint64_t n_verts = 0, vert_cap = 0; // padded
    DevBuf b_vblk, b_vflag, b_opos, b_onrm;
    bool vblk_raw = false; // a palette of more than kSkinRingMaxBones bones was loaded: every block raw from then on
    uint32_t n_entries = 0, entry_cap = 0; // bone tables: one entry per (surface, bone)
    DevBuf b_ib[3], b_palette;
    DevBuf b_bs, b_bs_w;  // blend-shape offsets (blocked f16) and weights
    uint64_t bs_used = 0; // shape blocks handed out
    uint32_t bs_w_used = 0;
    bool dirty = false; // the derived tables (SkinPlan) below are out of date
    DevBuf b_bone_slot, b_tiles, b_fold_node, b_fold_begin, b_fold_bone, b_fold_stale_idx, b_late_slot, b_stale_pos;
    DevBuf b_surf_of_slot, b_surf_bones; // per slot: the node's first skinned surface (FYX_NONE = none); per surface: its palette range
    uint32_t n_tiles = 0, n_fold = 0, n_late = 0, max_bones = 0;
    bool any_blend_shapes = false;

    bool is_skinned(uint32_t node) const { return node < skinned_node.size() && skinned_node[node]; }
    int32_t grow(fyx_ctx *c, uint32_t entries, uint64_t verts); // room for this many palette entries and (padded) vertices
    int32_t commit(fyx_ctx *c); // plan_skin, then the upload of the derived tables
    void topology_changed() { dirty = true; } // bone and mesh slots
    SkinArrays arrays() const;  // what the kernels read, from the buffers as they are now
    FoldArrays fold() const;
};

// The animations (fyx_anim_add, fyx_anim.inl): what the host reads of each animation and track, the blend groups, the
// records added since the last flush, and the device tables with the node CSR that plan_anim_nodes (fyx_anim_plan.hpp)
// derives from the tracks and the topology, which commit rebuilds when `dirty`.  Uploads wait for the first call that needs
// the device tables: thousands of animations (one per skeleton) arrive back to back at load time.
struct Animations {
    std::vector<AnimInfo> anims;
    std::vector<uint32_t> track_node, track_bk;      // per track, animation after animation: target node, binding | value_kind << 8
    std::vector<std::vector<uint32_t>> groups;       // sources of blend group g at [g - 1]
    uint32_t n_keys = 0;
    std::vector<fyx_curve_key> pend_keys;            // added since the last flush
    std::vector<AnimTrackDev> pend_tracks;
    std::vector<AnimStateDev> pend_state;
    DevBuf b_keys, b_tracks, b_state, b_hints, b_values, b_ok, b_bk, b_node_slot, b_node_begin, b_node_tracks;
    uint32_t n_nodes = 0; // of the node CSR
    bool dirty = true;    // the node CSR is out of date

    // Signals: the lists and capacities here; rings, queue heads and counts on the device once any animation has a signal
    std::vector<AnimSignals> sig;                   // per animation once signals_on
    bool signals_on = false, events_dirty = false;  // events_dirty: the device tables need relaying (commit)
    DevBuf b_sig, b_signals, b_events, b_drain; // b_drain: fyx_anim_take_events' header (2 words), then its events
    // Root motion: the settings per animation; the device records once any animation has had settings (they outlive them)
    std::vector<uint8_t> has_root;                  // per animation
    std::vector<fyx_root_motion_settings> root;     // per animation
    bool root_on = false, roots_dirty = false;
    uint32_t n_roots = 0, n_sig = 0, n_event_words = 0; // records in b_roots / b_sig, words in b_events
    DevBuf b_roots, b_rm, b_grm, b_group_begin, b_group_src; // b_grm: per group, BlendAnimations' output, then the final pose's
    uint64_t frames = 0;                            // fyx_animate calls that launched (a group is evaluated once one has)
    std::vector<uint64_t> group_born;               // `frames` when group g was made, at [g - 1]

    int32_t add(fyx_ctx *c, const fyx_animation_desc &d, uint32_t *out_id); // checks, then queues
    int32_t flush(fyx_ctx *c); // uploads the queue (the device tables grow, keeping the older animations' hints and time)
    int32_t commit(fyx_ctx *c); // flush, then plan_anim_nodes and its upload when dirty
    int32_t blend_group(fyx_ctx *c, uint32_t n, const uint32_t *ids, const float *weights, uint32_t *out_group);
    // v into `field` of device record i: the state of animation i, or track i
    template <class R, class F> int32_t write(fyx_ctx *c, uint32_t i, F R::*field, F v) const;
    void topology_changed() { dirty = true; } // target slots
    AnimArrays arrays() const; // what the kernels read, from the buffers as they are now
    int32_t download_events(fyx_ctx *c, std::vector<AnimSigDev> &d, std::vector<uint32_t> &ev) const;
    int32_t commit_events(fyx_ctx *c); // relays the signal tables (commit, when events_dirty)
    int32_t commit_roots(fyx_ctx *c);  // the root-motion tables (commit, when roots_dirty)
};

} // namespace

struct PeerState {
    DevBuf local;                          // this rank's exchange allocation (control block + 2 x F lists)
    void *mapped[kPeerMaxRanks] = {};      // the other ranks' allocations (cudaIpcOpenMemHandle)
    DevBuf cta_done;
    PinnedBuf h_counts;                    // [epoch & 1][2][rank][frustum] copy of the count table
    PeerParams pp{};
    bool ready = false;
};

struct fyx_ctx {
    int device = 0;
    cudaStream_t stream = nullptr; // own_stream, or the caller's stream from fyx_config (never destroyed here)
    Stream own_stream;
    std::string err;
    uint64_t launches = 0;

    // topology
    uint32_t n_nodes = 0, n_slots = 0, root = FYX_NONE, n_renderable = 0;
    std::vector<uint32_t> slot_of_node, node_of_slot, level_off;
    NodeArrays a{};
    DevBuf b_parent, b_flags, b_mask, b_gidx, b_G[3], b_la[3], b_wa[3], b_slot_of_node;
    SlotColumn L[3] = {SlotColumn(make_float4(1, 0, 0, 0)), SlotColumn(make_float4(0, 1, 0, 0)), SlotColumn(make_float4(0, 0, 1, 0))};
    bool have_topology = false, updated_once = false;
    SubforestPlan sf{};  // deep levels walked by one launch (fyx_internal.h); n_ctas = 0: one launch per level everywhere
    DevBuf b_sf_rng;
    // TransformBuilder's defaults (scene/transform.rs:176-200): the last position / rotation / scale sent for each node, and the
    // rarely changed rest of its Transform
    SlotColumn trs{fyx_trs{{0, 0, 0}, {0, 0, 0, 1}, {1, 1, 1}}};
    SlotColumn statics{fyx_transform_statics{{0, 0, 0, 1}, {1, 0, 0, 0, 1, 0, 0, 0, 1}, {0, 0, 0}, {0, 0, 0}, {0, 0, 0}, {0, 0, 0}}};
    std::array<SlotColumn *, 8> slot_columns() { return {&L[0], &L[1], &L[2], &trs, &statics, &bundle, &lod_range, &dyn.quads}; }

    // error word written by kernels
    DevBuf d_err;
    PinnedBuf h_err;

    // staging (host pinned + device)
    PinnedBuf h_stage;
    DevBuf d_stage;

    // cull outputs
    CullParams cp{};
    VisSlot vs[2];
    int cur = 0;      // slot written by the most recent cull
    int readable = 0; // slot fyx_get_visible reads
    uint64_t frame_counter = 0;

    // frame pipelining (FYX_FRAME_ASYNC): uploads on their own stream into alternating staging buffers,
    // read-backs on a third stream
    Stream copy_stream, d2h_stream;
    Stream fold_stream; // skinned-mesh fold + cull beside the palette / skinning kernels of asynchronous frames
    Event ev_levels_done, ev_fold_done;
    DevBuf d_stage_frame[2];
    Event ev_upload[2], ev_slot_free[2];
    bool slot_used[2] = {false, false};
    int upload_parity = 0;
    cudaEvent_t ev_levels_prev = nullptr; // the previous frame's "level kernels + fold + cull are done" event (its ev_cull), if it recorded one
    uint64_t launches_at_frame_end = ~0ull;

    Skinning skin;
    std::vector<uint32_t> dfs_rank; // optional: pre-order rank of every node in the reference's DFS (fyx_set_dfs_order); read through dfs_rank_of
    // surfaces per node (fyx_set_node_surfaces): host CSR by node, device table by slot (rebuilt when dirty)
    NodeRecords<uint2> ms_of_node{make_uint2(0u, 0u)}; // (first, count) into ms_bundle_h / ms_skin_h; count 0 = default single surface
    std::vector<uint32_t> ms_bundle_h, ms_skin_h;
    bool ms_dirty = false, have_ms = false;
    uint32_t ms_max = 0;                 // the most surfaces any node was given (bounds the shadow maps' bundle tables)
    DevBuf b_ms_range, b_ms_bundle, b_ms_skin;

    // timing
    Event ev[EV_COUNT];
    fyx_timings timings{};
    bool timings_pending = false; // an async frame's events have not been read yet
    bool stage_events_valid = false; // the last frame recorded the per-stage events (synchronous frames only)

    Animations anim; // N2 animation sampling

    // N4 LOD filter (fyx_drawprep.inl)
    SlotColumn lod_range{make_float2(NAN, NAN)}; // (begin, end); begin NaN = not a LOD object
    bool maybe_static_batch = false; // some node carries FYX_NODE_STATIC_BATCH: the cull runs un-fused, through the pruner table
    std::vector<fyx_observer> observers;

    // N4 light lists (fyx_drawprep.inl)
    DevBuf b_light[FYX_MAX_FRUSTA], b_light_ptrs, b_light_counts;
    PinnedBuf h_light_counts;
    std::vector<uint32_t> h_light[FYX_MAX_FRUSTA];
    uint32_t light_nf = 0;
    bool lights_valid = false;

    // N4 shadow casters (fyx_drawprep.inl): light-source records by node index, their device table by pool order, the maps
    NodeRecords<LightRec> light_src{LightRec{fyx_light_source{FYX_LIGHT_UNKNOWN, 0.f, 0.f}, 0.f}}; // kind FYX_LIGHT_UNKNOWN = no record
    NodeRecords<fyx_csm_options> csm_opts{kCsmDefault};
    bool light_table_dirty = false;
    uint32_t n_light_table = 0;
    DevBuf b_light_table;
    MapCull shadow_cull; // the last shadow cull: of one camera, or of the scene's observers
    // LOD filter and static-batch pruning of the camera culls and the many-map culls.  pr_node: by node index, kPrLod | kPrBatch
    // for a node with a LOD range / FYX_NODE_STATIC_BATCH (kept beside the device columns, so that a change is seen without
    // reading them back).  The pruner column is rebuilt by the first pruned cull after such a change (pr_dirty).
    NodeRecords<uint8_t> pr_node{uint8_t(0)};
    bool pr_dirty = true;
    uint32_t n_pruners = 0;
    std::vector<uint32_t> pr_level_off; // pruner ids per hierarchy level (pruners are numbered in slot order)
    DevBuf b_pr_col, b_pr_slot, b_pr_anc, b_pr_rows, b_pr_obs;

    // N4 scene observers (fyx_drawprep.inl): camera and reflection-probe records by node index, their device table (due
    // probes, then cameras, each in pool order; rebuilt when a record or the topology changes), the observer cull's outputs
    NodeRecords<CameraRec> cam_src{CameraRec{fyx_camera{0u, FYX_PROJECTION_NONE}, 0.f}}; // projection FYX_PROJECTION_NONE = no record
    NodeRecords<ProbeRec> probe_src{ProbeRec{fyx_reflection_probe{}, false}};            // present 0 = no record
    std::vector<uint32_t> ob_rec_node;          // node of each record of the device table
    bool obs_table_dirty = false;
    uint32_t n_ob_recs = 0;
    MapCull observer_cull; // a map per observer; its third small word is the light total
    DevBuf b_ob_recs, b_ob_table, b_ob_lcounts, b_ob_best, b_ob_lraw, b_ob_lights;
    PinnedBuf h_ob_table, h_ob_lights; // host copies of the table and the light lists
    uint32_t ob_light_total = 0;
    float ob_frame[2] = {0.f, 0.f}; // the frame size of the last observer cull
    uint64_t ob_epoch = 0;          // hier_epoch at the last observer cull

    // N4 shadow maps of the scene's observers (fyx_drawprep.inl): the map table and lists are the shadow cull's (`shadow_cull`);
    // the refs (observer, map), with the map-table kernel's scratch
    DevBuf b_ssh_refs, b_ssh_cand, b_ssh_hash, b_ssh_csm;
    PinnedBuf h_ssh_refs;
    uint32_t ssh_n_refs = 0;
    bool ssh_valid = false, ssh_on_host = false;
    uint64_t hier_epoch = 0; // counts fyx_set_topology and hierarchy updates: a table of another frame is refused

    // N3 draw-prep (fyx_drawprep.inl)
    bool instances_enabled = false, rank_on_device = false;
    uint32_t n_bundle_ids = 1;
    SlotColumn bundle{uint32_t(0)}; // bundle id per slot
    DevBuf b_rank_slot;
    PackScratch pack;
    InstPack inst[FYX_MAX_FRUSTA];

    DynBatches dyn; // Dynamic meshes and quad nodes

    // multi-GPU (fyx_comm.cu)
    void *comm = nullptr;
    int nranks = 1, rank = 0;
    Stream comm_stream; // the collective runs beside the palette / skinning kernels (highest priority)
    DevBuf b_counts_packed, b_counts_all;
    PinnedBuf h_counts_all; // nranks*FYX_MAX_FRUSTA
    bool want_peer = true, want_hostseg = true;
    unsigned peer_push_ctas = 96;
    bool exchange_built = false, hostseg_ready = false, hostseg_registered = false;
    uint32_t exchange_slots = 0, exch_nf_cap = 0;
    uint64_t exch_total_cap = 0, gather_epoch = 0;
    PeerState peer;
    HostSeg hostseg;
    Event ev_x0[2], ev_x1[2]; // timing of the exchange (per epoch parity)
    uint64_t x_epoch[2] = {0, 0};
    int x_slot[2] = {0, 0};
    Event ev_gath_read[2]; // private D2H copies of the gathered device lists (per epoch parity)
    bool gath_read_valid[2] = {false, false};
};

namespace {

int32_t fail(fyx_ctx *c, int32_t code, const char *fmt, ...)
{
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    if (c) c->err = buf;
    else g_create_error = buf;
    return code;
}

// the context's error message, for the checks of the planner headers
auto fail_of(fyx_ctx *c)
{
    return [c](int32_t code, const char *fmt, auto... args) { return fail(c, code, fmt, args...); };
}

#define CU(call)                                                                                         \
    do {                                                                                                 \
        cudaError_t e__ = (call);                                                                        \
        if (e__ != cudaSuccess)                                                                          \
            return fail(c, e__ == cudaErrorMemoryAllocation ? FYX_ERR_OUT_OF_MEMORY : FYX_ERR_CUDA,      \
                        "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), __FILE__, __LINE__);    \
    } while (0)

int32_t dev_ensure(fyx_ctx *c, DevBuf &b, size_t bytes, bool keep = false)
{
    if (bytes <= b.bytes) return FYX_OK;
    size_t nb = keep ? std::max(bytes, b.bytes + b.bytes / 2) : bytes;
    nb = (nb + 255) & ~size_t(255);
    DevBuf fresh;
    CU(fresh.alloc(nb));
    // growable tables are copied as a whole when they grow again: give their not-yet-written tail a defined value
    if (keep) CU(cudaMemsetAsync(fresh.p, 0, nb, c->stream));
    if (b.p) { // the old buffer stays valid until the stream has finished with it
        if (keep && b.bytes) CU(cudaMemcpyAsync(fresh.p, b.p, b.bytes, cudaMemcpyDeviceToDevice, c->stream));
        CU(cudaStreamSynchronize(c->stream));
    }
    b = std::move(fresh);
    return FYX_OK;
}

bool is_pinned(const void *p)
{
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return at.type == cudaMemoryTypeHost;
}

// Host → device staging of one or two arrays.  `direct` lets pinned caller memory be DMA'd without
// the bounce copy (only legal when the caller's buffer stays untouched until the next sync, i.e.
// inside fyx_render_prep).  Returns device pointers inside d_stage.
int32_t stage_to_device(fyx_ctx *c, const void *a0, size_t n0, const void *a1, size_t n1, bool direct, void **d0, void **d1)
{
    const size_t o1 = (n0 + 255) & ~size_t(255);
    const size_t total = o1 + ((n1 + 255) & ~size_t(255));
    int32_t rc = dev_ensure(c, c->d_stage, total);
    if (rc) return rc;
    char *dbase = c->d_stage.as<char>();
    const void *src[2] = {a0, a1};
    const size_t len[2] = {n0, n1};
    const size_t off[2] = {0, o1};
    bool need_bounce = false;
    for (int i = 0; i < 2; ++i)
        if (src[i] && len[i] && !(direct && is_pinned(src[i]))) need_bounce = true;
    if (need_bounce) {
        // the previous use of the bounce buffer must have drained, before it is refilled or replaced
        CU(cudaStreamSynchronize(c->stream));
        CU(c->h_stage.ensure(total));
    }
    for (int i = 0; i < 2; ++i) {
        if (!src[i] || !len[i]) continue;
        const void *from = src[i];
        if (!(direct && is_pinned(src[i]))) {
            memcpy(c->h_stage.as<char>() + off[i], src[i], len[i]);
            from = c->h_stage.as<char>() + off[i];
        }
        CU(cudaMemcpyAsync(dbase + off[i], from, len[i], cudaMemcpyHostToDevice, c->stream));
    }
    *d0 = (a0 && n0) ? dbase : nullptr;
    if (d1) *d1 = (a1 && n1) ? dbase + o1 : nullptr;
    return FYX_OK;
}

// `count` records of `words` 32-bit words from the host into the slots of their nodes (idx NULL = nodes 0..count-1)
int32_t scatter_words(fyx_ctx *c, uint32_t *dst, uint32_t words, uint32_t count, const uint32_t *idx, const void *values)
{
    void *d_v = nullptr, *d_i = nullptr;
    int32_t rc = stage_to_device(c, values, (size_t)count * words * 4, idx, idx ? (size_t)count * 4 : 0, false, &d_v, &d_i);
    if (rc) return rc;
    launch_scatter_words(c->stream, dst, words, count, static_cast<const uint32_t *>(d_i), static_cast<const uint32_t *>(d_v),
                         c->b_slot_of_node.as<uint32_t>(), c->n_nodes);
    c->launches++;
    CU(cudaGetLastError());
    return FYX_OK;
}

int32_t SlotColumn::ensure(fyx_ctx *c)
{
    if (live) return FYX_OK;
    int32_t rc = dev_ensure(c, buf, std::max<size_t>(c->n_slots, 1) * def.words * 4);
    if (rc) return rc;
    launch_permute_words(c->stream, buf.p, nullptr, nullptr, c->n_slots, def);
    c->launches++;
    live = true;
    return FYX_OK;
}

int32_t SlotColumn::carry(fyx_ctx *c, const uint32_t *old_of_new)
{
    if (!live) return FYX_OK;
    DevBuf fresh;
    int32_t rc = dev_ensure(c, fresh, std::max<size_t>(c->n_slots, 1) * def.words * 4);
    if (rc) return rc;
    launch_permute_words(c->stream, fresh.p, buf.p, old_of_new, c->n_slots, def);
    c->launches++;
    CU(cudaStreamSynchronize(c->stream)); // the old records are read before they are freed
    buf = std::move(fresh);
    return FYX_OK;
}

int32_t SlotColumn::scatter(fyx_ctx *c, uint32_t count, const uint32_t *idx, const void *values)
{
    int32_t rc = ensure(c);
    return rc ? rc : scatter_words(c, buf.as<uint32_t>(), def.words, count, idx, values);
}

} // namespace

template <class T> int32_t fyx::NodeRecords<T>::check(fyx_ctx *c, uint32_t count, const uint32_t *idx) const
{
    for (uint32_t e = 0; e < count; ++e) {
        const uint32_t node = idx ? idx[e] : e;
        if (node >= c->n_nodes) return fail(c, FYX_ERR_INVALID_ARGUMENT, "node %u out of range", node);
    }
    return FYX_OK;
}

namespace {

int32_t check_device_errors(fyx_ctx *c)
{
    // called right after a stream synchronisation; h_err was copied before it
    uint32_t &h_err = *c->h_err.as<uint32_t>();
    const uint32_t e = h_err;
    if (!e) return FYX_OK;
    h_err = 0;
    cudaMemsetAsync(c->d_err.p, 0, sizeof(uint32_t), c->stream);
    if (e & E_NOT_AFFINE)
        return fail(c, FYX_ERR_NOT_AFFINE, "a matrix with a bottom row other than (0,0,0,1) or a non-finite entry was skipped");
    if (e & E_BAD_BONE_INDEX) return fail(c, FYX_ERR_INVALID_ARGUMENT, "a vertex references a bone index >= n_bones");
    if (e & E_NONFINITE_VERTEX) return fail(c, FYX_ERR_INVALID_ARGUMENT, "a vertex position is not finite");
    if (e & E_PEER_TIMEOUT) return fail(c, FYX_ERR_NCCL, "the peer exchange of the visible lists timed out: a rank did not take part in the frame");
    if (e & E_SHADOW_LIST) return fail(c, FYX_ERR_CUDA, "internal: a pruned shadow map had more entries than its count pass found; its list is incomplete");
    return FYX_OK;
}

int32_t sync_and_check(fyx_ctx *c)
{
    CU(cudaMemcpyAsync(c->h_err.p, c->d_err.p, sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    CU(cudaGetLastError());
    return check_device_errors(c);
}

// The opening of every call that needs the scene: a context, and a topology (fyx_set_topology).  enter() also makes the
// context's device current; calls that check their arguments before they touch CUDA call topology_check() instead.
int32_t topology_check(fyx_ctx *c)
{
    if (!c) return FYX_ERR_INVALID_ARGUMENT;
    if (!c->have_topology) return fail(c, FYX_ERR_STATE, "fyx_set_topology has not been called");
    return FYX_OK;
}

int32_t enter(fyx_ctx *c)
{
    if (int32_t rc = topology_check(c)) return rc;
    CU(cudaSetDevice(c->device));
    return FYX_OK;
}

const uint32_t *dfs_rank_of(const fyx_ctx *c) { return valid_dfs_rank(c->dfs_rank, c->n_nodes); }

// a pruner mark (kPrLod / kPrBatch) of an alive node set or cleared; the pruner column is rebuilt when a mark changes
void pr_mark(fyx_ctx *c, uint32_t node, uint8_t bit, bool on)
{
    if (node >= c->n_nodes || c->slot_of_node[node] == FYX_NONE) return; // skipped by the scatter kernels too
    const uint8_t m = on ? (c->pr_node[node] | bit) : (c->pr_node[node] & ~bit);
    if (m == c->pr_node[node]) return;
    c->pr_node.set(node, m);
    c->pr_dirty = true;
}

void rebuild_node_arrays(fyx_ctx *c)
{
    NodeArrays &a = c->a;
    a.cap = c->n_slots;
    a.parent = c->b_parent.as<uint32_t>();
    a.flags = c->b_flags.as<uint32_t>();
    a.mask = c->b_mask.as<uint32_t>();
    a.gidx = c->b_gidx.as<uint32_t>();
    for (int i = 0; i < 3; ++i) {
        a.L[i] = c->L[i].buf.as<float4>();
        a.G[i] = c->b_G[i].as<float4>();
        a.la[i] = c->b_la[i].as<float2>();
        a.wa[i] = c->b_wa[i].as<float2>();
    }
}

int32_t prepare_cull(fyx_ctx *c, uint32_t nf, const fyx_frustum *fr, const uint32_t *cam_mask, const uint32_t *pass_flags)
{
    if (nf > FYX_MAX_FRUSTA) return fail(c, FYX_ERR_INVALID_ARGUMENT, "n_frusta %u > FYX_MAX_FRUSTA", nf);
    if (nf && !fr) return fail(c, FYX_ERR_INVALID_ARGUMENT, "frusta is NULL");
    const int slot = c->cur ^ 1;
    VisSlot &V = c->vs[slot];
    if (V.pending) return fail(c, FYX_ERR_STATE, "two pipelined frames are already in flight: call fyx_frame_wait first");
    c->cur = slot;
    c->cp.nf = (int)nf;
    c->cp.counts = V.d_counts.as<uint32_t>();
    c->cp.one = 1.0f;
    c->cp.negzero = -0.0f;
    for (uint32_t f = 0; f < nf; ++f) {
        to_dev_frustum(fr[f], cam_mask ? cam_mask[f] : 0xFFFFFFFFu, pass_flags ? pass_flags[f] : 0u, c->cp.f[f]);
        // worst case every alive node is visible (fyx_set_flags may turn any of them renderable)
        int32_t rc = dev_ensure(c, V.b_vis[f], sizeof(uint32_t) * std::max<size_t>(c->n_slots, 1));
        if (rc) return rc;
        c->cp.out[f] = V.b_vis[f].as<uint32_t>();
        c->cp.out_slot[f] = nullptr;
        if (c->instances_enabled) {
            rc = dev_ensure(c, V.b_vis_slot[f], sizeof(uint32_t) * std::max<size_t>(c->n_slots, 1));
            if (rc) return rc;
            c->cp.out_slot[f] = V.b_vis_slot[f].as<uint32_t>();
        }
    }
    V.have_slots = c->instances_enabled;
    for (auto &o : c->inst) o.valid = false;
    c->lights_valid = false;
    CU(cudaMemsetAsync(V.d_counts.p, 0, sizeof(uint32_t) * kCountStride * FYX_MAX_FRUSTA, c->stream));
    V.nf = nf;
    V.counts_on_host = V.lists_on_host = false;
    V.gathered = V.gathered_on_host = false;
    V.seg_published = V.seg_complete = V.own_in_seg = V.counts_all_known = V.host_copy_private = false;
    c->readable = slot;
    return FYX_OK;
}

// Hierarchy + boxes (+ fused cull): one launch per level (parents first), then the skinned-mesh fold.
// fold_on: stream for the skinned-mesh fold (+ cull of the skinned meshes); nullptr = the main stream, in order.  Another stream
// is given by asynchronous frames that go on to the palette / skinning kernels: those need the bones' matrices, not the meshes'
// boxes, so the (latency-bound) fold runs beside them; the caller joins the streams.
int32_t run_update(fyx_ctx *c, uint32_t update_flags, const CullParams *cull, cudaStream_t fold_on)
{
    const bool all = (update_flags & FYX_UPDATE_ALL) || !c->updated_once;
    const size_t nl = c->level_off.size() ? c->level_off.size() - 1 : 0;
    ++c->hier_epoch;
    const Skinning &sk = c->skin;
    if (sk.n_late) {
        launch_snapshot_bones(c->stream, c->a, sk.n_late, sk.b_late_slot.as<uint32_t>(), sk.b_stale_pos.as<float4>());
        c->launches++;
    }
    const size_t nl_wide = c->sf.n_ctas ? std::min<size_t>(nl, c->sf.first_level) : nl;
    for (size_t l = 0; l < nl_wide; ++l) {
        launch_update_level(c->stream, c->a, c->level_off[l], c->level_off[l + 1], all, cull);
        c->launches += (c->level_off[l + 1] > c->level_off[l]);
    }
    if (c->sf.n_ctas) { // the deep levels (small sub-trees: skeletons) in one launch
        launch_update_subforest(c->stream, c->a, c->sf, all, cull);
        c->launches++;
    }
    if (sk.n_fold) {
        if (fold_on) {
            CU(cudaEventRecord(c->ev_levels_done, c->stream));
            CU(cudaStreamWaitEvent(fold_on, c->ev_levels_done, 0));
        }
        launch_fold_bones(fold_on ? fold_on : c->stream, c->a, sk.fold(), cull);
        c->launches++;
        if (fold_on) CU(cudaEventRecord(c->ev_fold_done, fold_on));
    }
    c->updated_once = true;
    CU(cudaGetLastError());
    return FYX_OK;
}

// counts, then the lists sized by them, to pinned host memory (stream `s`, two synchronisations)
int32_t readback_visible(fyx_ctx *c, VisSlot &V, cudaStream_t s)
{
    const uint32_t nf = V.nf;
    if (!nf) return FYX_OK;
    if (!V.counts_on_host) {
        CU(cudaMemcpy2DAsync(V.h_counts.p, sizeof(uint32_t), V.d_counts.p, sizeof(uint32_t) * kCountStride, sizeof(uint32_t), nf,
                             cudaMemcpyDeviceToHost, s));
        CU(cudaStreamSynchronize(s));
        V.counts_on_host = true;
    }
    if (!V.lists_on_host) {
        for (uint32_t f = 0; f < nf; ++f) {
            const size_t n = V.h_counts.as<uint32_t>()[f];
            CU(V.h_vis[f].ensure(n * sizeof(uint32_t)));
            if (n) CU(cudaMemcpyAsync(V.h_vis[f].p, V.b_vis[f].p, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
        }
        CU(cudaStreamSynchronize(s));
        V.lists_on_host = true;
    }
    return FYX_OK;
}

} // namespace

// --------------------------------------------------------------------------------------------
// life cycle
// --------------------------------------------------------------------------------------------
extern "C" uint32_t fyx_abi_version(void) { return FYX_ABI_VERSION; }

extern "C" const char *fyx_last_error(const fyx_ctx *ctx) { return ctx ? ctx->err.c_str() : g_create_error.c_str(); }

extern "C" int32_t fyx_create(const fyx_config *cfg, fyx_ctx **out_ctx)
{
    fyx_ctx *c = nullptr; // for CU(): errors before the context exists go to the thread-local string
    if (!out_ctx) return fail(nullptr, FYX_ERR_INVALID_ARGUMENT, "out_ctx is NULL");
    *out_ctx = nullptr;
    int dev = -1;
    void *stream = nullptr;
    if (cfg) {
        if (cfg->struct_size < sizeof(fyx_config)) return fail(nullptr, FYX_ERR_INVALID_ARGUMENT, "fyx_config.struct_size too small");
        dev = cfg->device;
        stream = cfg->stream;
    }
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0)
        return fail(nullptr, FYX_ERR_CUDA, "no CUDA device available (%s): libfyrox_b200 has no CPU fallback",
                    e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
    if (dev < 0) CU(cudaGetDevice(&dev));
    if (dev >= count) return fail(nullptr, FYX_ERR_INVALID_ARGUMENT, "device %d out of range (%d devices)", dev, count);
    CU(cudaSetDevice(dev));
    cudaDeviceProp prop;
    CU(cudaGetDeviceProperties(&prop, dev));
    if (prop.major != 9 || prop.minor != 0)
        return fail(nullptr, FYX_ERR_CUDA, "device %d is sm_%d%d; this library ships sm_90a code only", dev, prop.major, prop.minor);

    // a failure below frees whatever was already made; CU() reports to fyx_last_error(NULL) because `c` stays NULL
    std::unique_ptr<fyx_ctx> ctx(new (std::nothrow) fyx_ctx());
    if (!ctx) return fail(nullptr, FYX_ERR_OUT_OF_MEMORY, "host allocation failed");
    ctx->device = dev;
    if (stream) {
        ctx->stream = static_cast<cudaStream_t>(stream);
    } else {
        CU(ctx->own_stream.create());
        ctx->stream = ctx->own_stream;
    }
    CU(ctx->d_err.alloc(sizeof(uint32_t)));
    CU(cudaMemset(ctx->d_err.p, 0, sizeof(uint32_t)));
    CU(ctx->h_err.ensure(sizeof(uint32_t)));
    *ctx->h_err.as<uint32_t>() = 0;
    for (VisSlot &V : ctx->vs) {
        CU(V.d_counts.alloc(sizeof(uint32_t) * kCountStride * FYX_MAX_FRUSTA));
        CU(cudaMemset(V.d_counts.p, 0, sizeof(uint32_t) * kCountStride * FYX_MAX_FRUSTA));
        CU(V.h_counts.ensure(sizeof(uint32_t) * FYX_MAX_FRUSTA));
        memset(V.h_counts.p, 0, sizeof(uint32_t) * FYX_MAX_FRUSTA);
        for (Event *ev : {&V.ev_cull, &V.ev_counts, &V.ev_done, &V.ev_gather, &V.ev_counts_all}) CU(ev->create(cudaEventDisableTiming));
    }
    for (int i = 0; i < 2; ++i) {
        CU(ctx->ev_gath_read[i].create(cudaEventDisableTiming));
        CU(ctx->ev_x0[i].create(cudaEventDefault));
        CU(ctx->ev_x1[i].create(cudaEventDefault));
    }
    CU(ctx->copy_stream.create());
    CU(ctx->d2h_stream.create());
    CU(ctx->fold_stream.create());
    CU(ctx->ev_levels_done.create(cudaEventDisableTiming));
    CU(ctx->ev_fold_done.create(cudaEventDisableTiming));
    for (int i = 0; i < 2; ++i) {
        CU(ctx->ev_upload[i].create(cudaEventDisableTiming));
        CU(ctx->ev_slot_free[i].create(cudaEventDisableTiming));
    }
    for (int i = 0; i < EV_COUNT; ++i) CU(ctx->ev[i].create(cudaEventDefault));
    *out_ctx = ctx.release();
    return FYX_OK;
}

static void fyx_comm_destroy_internal(fyx_ctx *c); // fyx_comm.inl
// DFS-pruning features (LOD filter, static batches): the cull cannot be fused into the level kernels (fyx_drawprep.inl)
static bool unfused_cull(const fyx_ctx *c, uint32_t nf);
static int32_t cull_unfused(fyx_ctx *c, uint32_t nf);
static int32_t cull_prune_prepare(fyx_ctx *c, uint32_t nf);
static int32_t animate_enqueue(fyx_ctx *c, float dt);  // fyx_anim.inl
static int32_t allgather_enqueue(fyx_ctx *c, VisSlot &V, cudaStream_t s);
static int32_t allgather_finish(fyx_ctx *c, VisSlot &V, cudaStream_t s);
static int32_t hostseg_publish(fyx_ctx *c, VisSlot &V, cudaStream_t s);
static int32_t resolve_counts(fyx_ctx *c, VisSlot &V);

extern "C" void fyx_destroy(fyx_ctx *c)
{
    if (!c) return;
    cudaSetDevice(c->device);
    // no stream may still use what the members free when they die
    for (cudaStream_t s : {c->stream, c->copy_stream.h, c->d2h_stream.h, c->fold_stream.h, c->comm_stream.h})
        if (s) cudaStreamSynchronize(s);
    fyx_comm_destroy_internal(c);
    delete c;
}

extern "C" int32_t fyx_sync(fyx_ctx *c)
{
    if (!c) return FYX_ERR_INVALID_ARGUMENT;
    return sync_and_check(c);
}

extern "C" void *fyx_host_alloc(size_t bytes)
{
    void *p = nullptr;
    if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault) != cudaSuccess) {
        cudaGetLastError();
        return nullptr;
    }
    return p;
}

extern "C" void fyx_host_free(void *p)
{
    if (p) cudaFreeHost(p);
}

extern "C" uint64_t fyx_kernel_launch_count(const fyx_ctx *c) { return c ? c->launches : 0; }

// --------------------------------------------------------------------------------------------
// host-side math (tiny, per frustum).  Built with -ffp-contract=off.
// --------------------------------------------------------------------------------------------
extern "C" int32_t fyx_frustum_from_view_projection_matrix(const float m[16], fyx_frustum *out)
{
    if (!m || !out) return FYX_ERR_INVALID_ARGUMENT;
    return frustum_from_view_projection(m, *out) ? FYX_OK : FYX_ERR_INVALID_ARGUMENT;
}

extern "C" void fyx_frustum_default(fyx_frustum *out)
{
    // Frustum::default: new_perspective(1.0, FRAC_PI_2, 0.01, 1024.0) (frustum.rs:32-43)
    float m[16] = {0};
    const float znear = 0.01f, zfar = 1024.0f;
    const float m22 = 1.0f / std::tan(1.57079632679489661923f / 2.0f);
    m[5] = m22;
    m[0] = m22 / 1.0f;
    m[10] = (zfar + znear) / (znear - zfar);
    m[14] = zfar * znear * 2.0f / (znear - zfar);
    m[11] = -1.0f;
    fyx_frustum_from_view_projection_matrix(m, out);
}

extern "C" void fyx_mat4_mul(const float a[16], const float b[16], float out[16]) { mat4_mul(a, b, out); }

// --------------------------------------------------------------------------------------------
// scene description
// --------------------------------------------------------------------------------------------
extern "C" int32_t fyx_set_topology(fyx_ctx *c, uint32_t capacity, uint32_t root, const uint32_t *parent, const uint32_t *flags,
                                    const uint32_t *render_mask, const float *local_aabb, const uint32_t *global_index)
{
    if (!c) return FYX_ERR_INVALID_ARGUMENT;
    if (capacity && !parent) return fail(c, FYX_ERR_INVALID_ARGUMENT, "parent is NULL");
    if (capacity == FYX_NONE) return fail(c, FYX_ERR_INVALID_ARGUMENT, "capacity too large");
    CU(cudaSetDevice(c->device));
    SlotPlan plan = plan_slots(capacity, parent, flags);
    if (plan.cycle_node != FYX_NONE) return fail(c, FYX_ERR_TOPOLOGY, "cycle in parent[] through node %u", plan.cycle_node);
    const char *env = getenv("FYX_SUBFOREST"); // 1 forces the sub-forest plan on, 0 off
    const SubforestLayout sf = plan_subforest(plan, (env && *env) ? atoi(env) : -1);
    const uint32_t n_slots = plan.n_slots();

    // slot-ordered host columns
    const uint32_t def_flags = FYX_NODE_VISIBILITY | FYX_NODE_ENABLED | FYX_NODE_FRUSTUM_CULLING | FYX_NODE_CAST_SHADOWS | FYX_NODE_ALIVE;
    std::vector<uint32_t> h_flags(n_slots), h_mask(n_slots), h_gidx(n_slots);
    std::vector<float2> h_la[3];
    for (auto &v : h_la) v.resize(n_slots);
    std::vector<uint32_t> static_batch; // nodes with FYX_NODE_STATIC_BATCH
    uint32_t n_renderable = 0;
    for (uint32_t s = 0; s < n_slots; ++s) {
        const uint32_t i = plan.node_of_slot[s];
        uint32_t f = (flags ? (flags[i] & FYX_NODE_INPUT_MASK) : def_flags) | F_DIRTY_SELF;
        if (i == root) f |= F_ROOT;
        if (c->skin.is_skinned(i)) f |= F_SKINNED;
        h_flags[s] = f;
        n_renderable += (f & FYX_NODE_RENDERABLE) ? 1u : 0u;
        if (f & FYX_NODE_STATIC_BATCH) static_batch.push_back(i);
        h_mask[s] = render_mask ? render_mask[i] : 0xFFFFFFFFu;
        h_gidx[s] = global_index ? global_index[i] : i;
        if (local_aabb) {
            const float *b = local_aabb + 6 * (size_t)i;
            h_la[0][s] = make_float2(b[0], b[3]);
            h_la[1][s] = make_float2(b[1], b[4]);
            h_la[2][s] = make_float2(b[2], b[5]);
        } else { // AxisAlignedBoundingBox::unit(), scene/base.rs:733-735
            h_la[0][s] = h_la[1][s] = h_la[2][s] = make_float2(-0.5f, 0.5f);
        }
    }

    // Per-node data that is NOT an argument of this call survives it: the slot columns (local matrices, TRS records, transform
    // statics, bundle ids and LOD ranges) of every node that was alive before and still is are carried from their old slot to
    // the new one on the device (nodes that were not alive start from the defaults).  old_of_new[s] = the old slot.
    const bool carry = c->have_topology && c->n_slots > 0 && n_slots > 0;
    DevBuf b_map;
    int32_t rc;
    if (carry) {
        std::vector<uint32_t> old_of_new(n_slots, FYX_NONE);
        for (uint32_t s = 0; s < n_slots; ++s) {
            const uint32_t i = plan.node_of_slot[s];
            if (i < c->n_nodes && c->slot_of_node[i] != FYX_NONE) old_of_new[s] = c->slot_of_node[i];
        }
        if ((rc = dev_ensure(c, b_map, (size_t)n_slots * 4))) return rc;
        CU(cudaStreamSynchronize(c->stream));
        CU(cudaMemcpy(b_map.p, old_of_new.data(), (size_t)n_slots * 4, cudaMemcpyHostToDevice));
    }
    c->n_slots = n_slots;
    for (SlotColumn *col : c->slot_columns()) {
        if (!carry) col->live = false; // nothing to carry over (first topology, or one side empty): the column starts afresh
        else if ((rc = col->carry(c, b_map.as<uint32_t>()))) return rc;
    }
    if (!carry) c->n_bundle_ids = 1;

    // device columns.  Everything is allocated before the fills below are launched: the planes the level kernels stream side by
    // side stay adjacent in allocation order (with a fill launched between them, k_update_level measured ~1% slower on an
    // H100 80GB HBM3 at a 400 W power limit).
    const size_t n = std::max<uint32_t>(n_slots, 1);
    if ((rc = dev_ensure(c, c->b_parent, n * 4))) return rc;
    if ((rc = dev_ensure(c, c->b_flags, n * 4))) return rc;
    if ((rc = dev_ensure(c, c->b_mask, n * 4))) return rc;
    if ((rc = dev_ensure(c, c->b_gidx, n * 4))) return rc;
    if ((rc = dev_ensure(c, c->b_slot_of_node, std::max<size_t>(capacity, 1) * 4))) return rc;
    for (int k = 0; k < 3; ++k) {
        if ((rc = dev_ensure(c, c->L[k].buf, n * sizeof(float4)))) return rc; // filled by L[k].ensure below unless carried
        if ((rc = dev_ensure(c, c->b_G[k], n * sizeof(float4)))) return rc;
        if ((rc = dev_ensure(c, c->b_la[k], n * sizeof(float2)))) return rc;
        if ((rc = dev_ensure(c, c->b_wa[k], n * sizeof(float2)))) return rc;
    }
    CU(cudaStreamSynchronize(c->stream));
    if (n_slots) {
        CU(cudaMemcpy(c->b_parent.p, plan.parent.data(), n_slots * 4, cudaMemcpyHostToDevice));
        CU(cudaMemcpy(c->b_flags.p, h_flags.data(), n_slots * 4, cudaMemcpyHostToDevice));
        CU(cudaMemcpy(c->b_mask.p, h_mask.data(), n_slots * 4, cudaMemcpyHostToDevice));
        CU(cudaMemcpy(c->b_gidx.p, h_gidx.data(), n_slots * 4, cudaMemcpyHostToDevice));
        for (int k = 0; k < 3; ++k) CU(cudaMemcpy(c->b_la[k].p, h_la[k].data(), n_slots * sizeof(float2), cudaMemcpyHostToDevice));
    }
    if (capacity) CU(cudaMemcpy(c->b_slot_of_node.p, plan.slot_of_node.data(), (size_t)capacity * 4, cudaMemcpyHostToDevice));
    c->sf = SubforestPlan{};
    if (sf.n_ctas()) {
        static_assert(sizeof(SfRange) == sizeof(uint2), "a sub-forest range is the uint2 the kernel reads");
        if ((rc = dev_ensure(c, c->b_sf_rng, sf.rng.size() * sizeof(uint2)))) return rc;
        CU(cudaMemcpy(c->b_sf_rng.p, sf.rng.data(), sf.rng.size() * sizeof(uint2), cudaMemcpyHostToDevice));
        c->sf.n_ctas = sf.n_ctas();
        c->sf.n_levels = sf.n_levels;
        c->sf.first_level = sf.first_level;
        c->sf.rng = c->b_sf_rng.as<uint2>();
    }
    // local rows are always there; global matrices start as identity rows (the local rows' default), world boxes as
    // AABB::default()
    for (int k = 0; k < 3; ++k) {
        if ((rc = c->L[k].ensure(c))) return rc;
        launch_permute_words(c->stream, c->b_G[k].p, nullptr, nullptr, n_slots, c->L[k].def);
        launch_permute_words(c->stream, c->b_wa[k].p, nullptr, nullptr, n_slots, WordRecord(make_float2(3.402823466e38f, -3.402823466e38f)));
        c->launches += 2;
    }

    const bool same_capacity = c->have_topology && capacity == c->n_nodes;
    const std::vector<uint32_t> old_slot_of_node = std::move(c->slot_of_node);
    c->slot_of_node = std::move(plan.slot_of_node);
    c->node_of_slot = std::move(plan.node_of_slot);
    c->level_off = std::move(plan.level_off);
    c->n_nodes = capacity;
    c->root = root;
    c->n_renderable = n_renderable;
    c->maybe_static_batch = !static_batch.empty();
    c->have_topology = true;
    c->updated_once = false;
    rebuild_node_arrays(c);

    // the other owners of per-node data
    const std::vector<uint32_t> &new_slot_of_node = c->slot_of_node;
    c->light_src.topology_changed(old_slot_of_node, new_slot_of_node);
    c->csm_opts.topology_changed(old_slot_of_node, new_slot_of_node);
    c->cam_src.topology_changed(old_slot_of_node, new_slot_of_node);
    c->probe_src.topology_changed(old_slot_of_node, new_slot_of_node);
    c->ms_of_node.topology_changed(old_slot_of_node, new_slot_of_node);
    // a pruner mark keeps its LOD bit (as the LOD range column does); static batches come from the new flags
    c->pr_node.topology_changed(old_slot_of_node, new_slot_of_node, [](uint8_t &m) { m &= kPrLod; });
    for (uint32_t i : static_batch) pr_mark(c, i, kPrBatch, true);
    c->shadow_cull.topology_changed();
    c->observer_cull.topology_changed();
    c->dyn.topology_changed(old_slot_of_node, new_slot_of_node);
    c->skin.topology_changed();
    c->anim.topology_changed();

    // the tables derived from them, which address nodes by slot
    c->light_table_dirty = true;
    c->obs_table_dirty = true;
    c->ms_dirty = c->have_ms;
    c->pr_dirty = true;
    if (!same_capacity) c->dfs_rank.clear(); // indexed by node: stays valid while the pool capacity does
    c->rank_on_device = false;
    ++c->hier_epoch;
    return FYX_OK;
}

extern "C" int32_t fyx_set_dfs_order(fyx_ctx *c, uint32_t capacity, const uint32_t *preorder_rank)
{
    if (int32_t rc = topology_check(c)) return rc;
    if (preorder_rank && capacity != c->n_nodes) return fail(c, FYX_ERR_INVALID_ARGUMENT, "capacity %u != topology capacity %u", capacity, c->n_nodes);
    if (preorder_rank) c->dfs_rank.assign(preorder_rank, preorder_rank + capacity);
    else c->dfs_rank.clear();
    c->rank_on_device = false;
    c->skin.dirty = true; // late bones
    c->dyn.invalidate();
    return FYX_OK;
}

// The forms of changed local transforms: 4x4 matrices, TRS records, or rotations alone (the last position and scale stay)
enum LocalsForm { LOCALS_M16, LOCALS_TRS, LOCALS_ROT };

// `count` changed local transforms, already on the device (d_idx NULL = nodes 0..count-1), into their nodes' slots on stream `s`.
// The TRS forms go through the TRS column, which keeps the parts a rotation alone does not change.
static int32_t scatter_locals(fyx_ctx *c, cudaStream_t s, LocalsForm form, uint32_t count, const uint32_t *d_idx, const void *d_payload)
{
    if (form == LOCALS_M16) {
        launch_scatter_locals(s, c->a, count, d_idx, static_cast<const float *>(d_payload), c->b_slot_of_node.as<uint32_t>(), c->n_nodes,
                              c->d_err.as<uint32_t>());
    } else {
        int32_t rc = c->trs.ensure(c);
        if (rc) return rc;
        launch_scatter_trs(s, c->a, count, d_idx, d_payload, form == LOCALS_ROT, c->trs.buf.as<fyx_trs>(),
                           c->statics.live ? c->statics.buf.as<fyx_transform_statics>() : nullptr, c->b_slot_of_node.as<uint32_t>(), c->n_nodes,
                           c->d_err.as<uint32_t>());
    }
    c->launches++;
    CU(cudaGetLastError());
    return FYX_OK;
}

extern "C" int32_t fyx_set_local_matrices(fyx_ctx *c, uint32_t count, const uint32_t *idx, const float *m16)
{
    if (int32_t rc = topology_check(c)) return rc;
    if (!count) return FYX_OK;
    if (!m16) return fail(c, FYX_ERR_INVALID_ARGUMENT, "m16 is NULL");
    CU(cudaSetDevice(c->device));
    void *d_m = nullptr, *d_i = nullptr;
    int32_t rc = stage_to_device(c, m16, (size_t)count * 64, idx, idx ? (size_t)count * 4 : 0, false, &d_m, &d_i);
    return rc ? rc : scatter_locals(c, c->stream, LOCALS_M16, count, static_cast<const uint32_t *>(d_i), d_m);
}

extern "C" int32_t fyx_set_local_rotations(fyx_ctx *c, uint32_t count, const uint32_t *idx, const float *quat_ijkw)
{
    if (int32_t rc = topology_check(c)) return rc;
    if (!count) return FYX_OK;
    if (!quat_ijkw) return fail(c, FYX_ERR_INVALID_ARGUMENT, "rotations are NULL");
    CU(cudaSetDevice(c->device));
    void *d_q = nullptr, *d_i = nullptr;
    int32_t rc = stage_to_device(c, quat_ijkw, (size_t)count * 16, idx, idx ? (size_t)count * 4 : 0, false, &d_q, &d_i);
    return rc ? rc : scatter_locals(c, c->stream, LOCALS_ROT, count, static_cast<const uint32_t *>(d_i), d_q);
}

extern "C" int32_t fyx_set_local_trs(fyx_ctx *c, uint32_t count, const uint32_t *idx, const fyx_trs *trs)
{
    if (int32_t rc = topology_check(c)) return rc;
    if (!count) return FYX_OK;
    if (!trs) return fail(c, FYX_ERR_INVALID_ARGUMENT, "trs is NULL");
    CU(cudaSetDevice(c->device));
    void *d_t = nullptr, *d_i = nullptr;
    int32_t rc = stage_to_device(c, trs, (size_t)count * sizeof(fyx_trs), idx, idx ? (size_t)count * 4 : 0, false, &d_t, &d_i);
    return rc ? rc : scatter_locals(c, c->stream, LOCALS_TRS, count, static_cast<const uint32_t *>(d_i), d_t);
}

extern "C" int32_t fyx_set_transform_statics(fyx_ctx *c, uint32_t count, const uint32_t *idx, const fyx_transform_statics *statics)
{
    if (int32_t rc = topology_check(c)) return rc;
    if (!count) return FYX_OK;
    if (!statics) return fail(c, FYX_ERR_INVALID_ARGUMENT, "statics is NULL");
    CU(cudaSetDevice(c->device));
    return c->statics.scatter(c, count, idx, statics);
}

extern "C" int32_t fyx_set_flags(fyx_ctx *c, uint32_t count, const uint32_t *idx, const uint32_t *flags)
{
    if (int32_t rc = topology_check(c)) return rc;
    if (!count) return FYX_OK;
    if (!flags) return fail(c, FYX_ERR_INVALID_ARGUMENT, "values are NULL");
    for (uint32_t i = 0; i < count; ++i)
        if (flags[i] & FYX_NODE_STATIC_BATCH) c->maybe_static_batch = true; // conservative: stays on until the next topology
    CU(cudaSetDevice(c->device));
    void *d_v = nullptr, *d_i = nullptr;
    int32_t rc = stage_to_device(c, flags, (size_t)count * 4, idx, idx ? (size_t)count * 4 : 0, false, &d_v, &d_i);
    if (rc) return rc;
    for (uint32_t i = 0; i < count; ++i) // the pruner marks, as k_scatter_flags resolves the nodes
        pr_mark(c, idx ? idx[i] : i, kPrBatch, (flags[i] & FYX_NODE_STATIC_BATCH) != 0);
    launch_scatter_flags(c->stream, c->a.flags, count, static_cast<const uint32_t *>(d_i), static_cast<const uint32_t *>(d_v),
                         c->b_slot_of_node.as<uint32_t>(), c->n_nodes);
    c->launches++;
    CU(cudaGetLastError());
    return FYX_OK;
}

extern "C" int32_t fyx_set_render_masks(fyx_ctx *c, uint32_t count, const uint32_t *idx, const uint32_t *mask)
{
    if (int32_t rc = topology_check(c)) return rc;
    if (!count) return FYX_OK;
    if (!mask) return fail(c, FYX_ERR_INVALID_ARGUMENT, "values are NULL");
    CU(cudaSetDevice(c->device));
    return scatter_words(c, c->a.mask, 1, count, idx, mask);
}

extern "C" int32_t fyx_set_local_aabbs(fyx_ctx *c, uint32_t count, const uint32_t *idx, const float *aabb)
{
    if (int32_t rc = topology_check(c)) return rc;
    if (!count) return FYX_OK;
    if (!aabb) return fail(c, FYX_ERR_INVALID_ARGUMENT, "aabb is NULL");
    CU(cudaSetDevice(c->device));
    void *d_v = nullptr, *d_i = nullptr;
    int32_t rc = stage_to_device(c, aabb, (size_t)count * 24, idx, idx ? (size_t)count * 4 : 0, false, &d_v, &d_i);
    if (rc) return rc;
    launch_scatter_aabbs(c->stream, c->a, count, static_cast<const uint32_t *>(d_i), static_cast<const float *>(d_v),
                         c->b_slot_of_node.as<uint32_t>(), c->n_nodes);
    c->launches++;
    CU(cudaGetLastError());
    return FYX_OK;
}

// --------------------------------------------------------------------------------------------
// skinned surfaces
// --------------------------------------------------------------------------------------------
namespace {

int32_t Skinning::grow(fyx_ctx *c, uint32_t entries, uint64_t verts)
{
    int32_t rc;
    if (entries > entry_cap) {
        for (int k = 0; k < 3; ++k)
            if ((rc = dev_ensure(c, b_ib[k], (size_t)entries * 16, true))) return rc;
        if ((rc = dev_ensure(c, b_palette, (size_t)entries * 64, true))) return rc;
        entry_cap = (uint32_t)std::min<size_t>({b_ib[0].bytes / 16, b_ib[1].bytes / 16, b_ib[2].bytes / 16, b_palette.bytes / 64});
    }
    if (verts > vert_cap) {
        const uint64_t blocks = (verts + 127) / 128 + 1; // 128-vertex blocks of 11 x 512 B
        if ((rc = dev_ensure(c, b_vblk, blocks * kVblkStride * sizeof(float4), true))) return rc;
        if ((rc = dev_ensure(c, b_vflag, blocks, true))) return rc;
        if ((rc = dev_ensure(c, b_opos, verts * 12, true))) return rc;
        if ((rc = dev_ensure(c, b_onrm, verts * 12, true))) return rc;
        vert_cap = std::min<uint64_t>({(b_vblk.bytes / (kVblkStride * sizeof(float4)) - 1) * 128, (b_vflag.bytes - 1) * 128, b_opos.bytes / 12,
                                       b_onrm.bytes / 12});
    }
    return FYX_OK;
}

SkinArrays Skinning::arrays() const
{
    return SkinArrays{n_entries, b_bone_slot.as<uint32_t>(), {b_ib[0].as<float4>(), b_ib[1].as<float4>(), b_ib[2].as<float4>()}, b_palette.as<float>(),
                      b_vblk.as<float4>(), b_opos.as<float>(), b_onrm.as<float>(), b_bs.as<uint2>(), b_bs_w.as<float>()};
}

FoldArrays Skinning::fold() const
{
    return FoldArrays{n_fold, b_fold_node.as<uint32_t>(), b_fold_begin.as<uint32_t>(), b_fold_bone.as<uint32_t>(),
                      n_late ? b_fold_stale_idx.as<uint32_t>() : nullptr, n_late ? b_stale_pos.as<float4>() : nullptr};
}

// `v` into `b`, sized for at least one element; the stream has finished reading `b`
template <class T> int32_t upload(fyx_ctx *c, DevBuf &b, const std::vector<T> &v)
{
    if (int32_t rc = dev_ensure(c, b, std::max<size_t>(v.size(), 1) * sizeof(T))) return rc;
    if (!v.empty()) CU(cudaMemcpy(b.p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
    return FYX_OK;
}

int32_t Skinning::commit(fyx_ctx *c)
{
    if (!dirty) return FYX_OK;
    if (int32_t rc = topology_check(c)) return rc;
    const SkinPlan p = plan_skin(surfaces, c->slot_of_node, c->n_slots, dfs_rank_of(c));
    static_assert(sizeof(SurfBones) == sizeof(uint2), "a palette range is the uint2 the bone-block kernels read");
    CU(cudaStreamSynchronize(c->stream));
    int32_t rc;
    if ((rc = upload(c, b_bone_slot, p.bone_slot)) || (rc = upload(c, b_tiles, p.tiles)) || (rc = upload(c, b_fold_node, p.fold_node)) ||
        (rc = upload(c, b_fold_begin, p.fold_begin)) || (rc = upload(c, b_fold_bone, p.fold_bone)) ||
        (rc = upload(c, b_surf_of_slot, p.surf_of_slot)) || (rc = upload(c, b_surf_bones, p.surf_bones)))
        return rc;
    if (!p.late_slot.empty()) {
        if ((rc = upload(c, b_fold_stale_idx, p.stale_idx)) || (rc = upload(c, b_late_slot, p.late_slot))) return rc;
        if ((rc = dev_ensure(c, b_stale_pos, p.late_slot.size() * sizeof(float4)))) return rc;
    }
    launch_tile_vcode(c->stream, b_tiles.as<SkinTile>(), (uint32_t)p.tiles.size(), b_vflag.as<uint8_t>());
    n_tiles = (uint32_t)p.tiles.size();
    n_fold = (uint32_t)p.fold_node.size();
    n_late = (uint32_t)p.late_slot.size();
    max_bones = p.max_bones;
    any_blend_shapes = p.any_blend_shapes;
    dirty = false;
    return FYX_OK;
}

} // namespace

extern "C" int32_t fyx_add_skinned_surface(fyx_ctx *c, uint32_t mesh_node, uint32_t n_bones, const uint32_t *bone_nodes,
                                           const float *inv_bind, uint32_t n_verts, const void *verts,
                                           const fyx_vertex_layout *layout, uint32_t *out_id)
{
    if (int32_t rc = topology_check(c)) return rc;
    if (n_bones > FYX_MAX_BONES) return fail(c, FYX_ERR_INVALID_ARGUMENT, "n_bones %u > %u", n_bones, FYX_MAX_BONES);
    if (n_bones && (!bone_nodes || !inv_bind)) return fail(c, FYX_ERR_INVALID_ARGUMENT, "bone arrays are NULL");
    if (n_verts && (!verts || !layout)) return fail(c, FYX_ERR_INVALID_ARGUMENT, "verts/layout are NULL");
    if (n_verts && !n_bones) return fail(c, FYX_ERR_INVALID_ARGUMENT, "a skinned surface needs at least one bone");
    if (n_verts) {
        const fyx_vertex_layout &l = *layout;
        if (l.stride % 4 || l.position_offset % 4 || l.normal_offset % 4 || l.bone_weights_offset % 4 || l.bone_indices_offset % 4)
            return fail(c, FYX_ERR_UNSUPPORTED, "vertex stride and attribute offsets must be multiples of 4");
        if (l.position_offset + 12 > l.stride || l.normal_offset + 12 > l.stride || l.bone_weights_offset + 16 > l.stride ||
            l.bone_indices_offset + 4 > l.stride)
            return fail(c, FYX_ERR_INVALID_ARGUMENT, "vertex attribute outside the vertex");
    }
    CU(cudaSetDevice(c->device));
    Skinning &sk = c->skin;
    SkinSurface sf;
    sf.mesh_node = mesh_node;
    sf.bones.assign(bone_nodes, bone_nodes + n_bones);
    sf.bone_off = sk.n_entries;
    sf.n_verts = n_verts;
    sf.vert_off = sk.n_verts;
    const uint64_t padded = ((uint64_t)n_verts + 3) & ~uint64_t(3);
    int32_t rc;
    if ((rc = sk.grow(c, sk.n_entries + n_bones, sk.n_verts + padded))) return rc;
    if (n_bones) {
        void *d_m = nullptr;
        if ((rc = stage_to_device(c, inv_bind, (size_t)n_bones * 64, nullptr, 0, false, &d_m, nullptr))) return rc;
        launch_ib_rows(c->stream, n_bones, static_cast<const float *>(d_m), sk.b_ib[0].as<float4>() + sf.bone_off,
                       sk.b_ib[1].as<float4>() + sf.bone_off, sk.b_ib[2].as<float4>() + sf.bone_off, c->d_err.as<uint32_t>());
        c->launches++;
    }
    if (n_verts) {
        void *d_v = nullptr;
        if ((rc = stage_to_device(c, verts, (size_t)n_verts * layout->stride, nullptr, 0, false, &d_v, nullptr))) return rc;
        if (n_bones > kSkinRingMaxBones && !sk.vblk_raw) { // k_skin's register-load form reads raw blocks
            launch_vdecode_all(c->stream, sk.b_vblk.as<float4>(), sk.b_vflag.as<uint8_t>(), (sk.n_verts + 127) / 128);
            sk.vblk_raw = true;
        }
        launch_deinterleave(c->stream, n_verts, static_cast<const unsigned char *>(d_v), *layout, n_bones, sk.b_vblk.as<float4>(),
                            sk.b_vflag.as<uint8_t>(), !sk.vblk_raw, sf.vert_off, c->d_err.as<uint32_t>());
        c->launches++;
    }
    CU(cudaGetLastError());
    sk.n_entries += n_bones;
    sk.n_verts += padded;
    if (n_bones && mesh_node < c->n_nodes && !sk.is_skinned(mesh_node)) {
        if (sk.skinned_node.size() < c->n_nodes) sk.skinned_node.resize(c->n_nodes, 0);
        sk.skinned_node[mesh_node] = 1;
        const uint32_t slot = c->slot_of_node[mesh_node];
        if (slot != FYX_NONE) {
            launch_or_u32(c->stream, c->a.flags + slot, F_SKINNED | F_DIRTY_SELF);
            c->launches++;
        }
    }
    if (out_id) *out_id = (uint32_t)sk.surfaces.size();
    sk.surfaces.push_back(std::move(sf));
    sk.dirty = true;
    return FYX_OK;
}

// N4: blend shapes of a surface (BlendShapesContainer, scene/mesh/surface.rs:92-218) and their weights (Mesh::blend_shapes,
// scene/mesh/mod.rs:449-456; the renderer passes weight / 100, :794-798)
extern "C" int32_t fyx_set_blend_shapes(fyx_ctx *c, uint32_t sid, uint32_t n_shapes, const void *records, uint32_t layer_stride, const float *weights)
{
    if (!c) return FYX_ERR_INVALID_ARGUMENT;
    Skinning &sk = c->skin;
    if (sid >= sk.surfaces.size()) return fail(c, FYX_ERR_INVALID_ARGUMENT, "surface id %u out of range", sid);
    if (n_shapes > FYX_MAX_BLEND_SHAPES) return fail(c, FYX_ERR_INVALID_ARGUMENT, "n_shapes %u > %u", n_shapes, FYX_MAX_BLEND_SHAPES);
    SkinSurface &sf = sk.surfaces[sid];
    if (n_shapes && !records) return fail(c, FYX_ERR_INVALID_ARGUMENT, "records are NULL");
    if (n_shapes && layer_stride < sf.n_verts) return fail(c, FYX_ERR_INVALID_ARGUMENT, "layer_stride %u < the surface's %u vertices", layer_stride, sf.n_verts);
    CU(cudaSetDevice(c->device));
    sk.dirty = true;
    if (!n_shapes || !sf.n_verts) {
        sf.n_shapes = 0;
        return FYX_OK;
    }
    const uint32_t bs_blocks = (sf.n_verts + 127u) / 128u;
    const uint64_t need = (uint64_t)n_shapes * bs_blocks;
    if (need > 0xFFFFFFFFull) return fail(c, FYX_ERR_INVALID_ARGUMENT, "too much blend-shape data");
    int32_t rc;
    if (need > sf.bs_cap) { // a new region at the end (an earlier, smaller region of this surface is abandoned)
        if (sk.bs_used + need > 0xFFFFFFFFull) return fail(c, FYX_ERR_OUT_OF_MEMORY, "blend-shape storage exhausted");
        if ((rc = dev_ensure(c, sk.b_bs, (sk.bs_used + need) * kBsBlockU2 * sizeof(uint2), true))) return rc;
        sf.bs_off = sk.bs_used;
        sf.bs_cap = (uint32_t)need;
        sk.bs_used += need;
    }
    if (n_shapes > sf.w_cap) {
        if ((rc = dev_ensure(c, sk.b_bs_w, (size_t)(sk.bs_w_used + n_shapes) * sizeof(float), true))) return rc;
        sf.w_off = sk.bs_w_used;
        sf.w_cap = n_shapes;
        sk.bs_w_used += n_shapes;
    }
    sf.n_shapes = n_shapes;
    sf.bs_blocks = bs_blocks;
    std::vector<float> w(n_shapes);
    for (uint32_t i = 0; i < n_shapes; ++i) w[i] = (weights ? weights[i] : 100.0f) / 100.0f; // bs.weight / 100.0 (mesh/mod.rs:797)
    void *d_rec = nullptr, *d_w = nullptr;
    if ((rc = stage_to_device(c, records, (size_t)n_shapes * layer_stride * 18, w.data(), (size_t)n_shapes * 4, false, &d_rec, &d_w))) return rc;
    launch_bs_layout(c->stream, sf.n_verts, n_shapes, layer_stride, static_cast<const uint16_t *>(d_rec), sk.b_bs.as<uint2>() + sf.bs_off * kBsBlockU2, bs_blocks);
    c->launches++;
    CU(cudaMemcpyAsync(sk.b_bs_w.as<float>() + sf.w_off, d_w, (size_t)n_shapes * 4, cudaMemcpyDeviceToDevice, c->stream));
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(c->stream)); // `w` and the staging buffer are free again
    return FYX_OK;
}

extern "C" int32_t fyx_set_blend_shape_weights(fyx_ctx *c, uint32_t sid, uint32_t n, const float *weights)
{
    if (!c) return FYX_ERR_INVALID_ARGUMENT;
    Skinning &sk = c->skin;
    if (sid >= sk.surfaces.size()) return fail(c, FYX_ERR_INVALID_ARGUMENT, "surface id %u out of range", sid);
    SkinSurface &sf = sk.surfaces[sid];
    if (n != sf.n_shapes) return fail(c, FYX_ERR_INVALID_ARGUMENT, "the surface has %u blend shapes, %u weights given", sf.n_shapes, n);
    if (!n) return FYX_OK;
    if (!weights) return fail(c, FYX_ERR_INVALID_ARGUMENT, "weights are NULL");
    CU(cudaSetDevice(c->device));
    std::vector<float> w(n);
    for (uint32_t i = 0; i < n; ++i) w[i] = weights[i] / 100.0f;
    void *d_w = nullptr;
    int32_t rc = stage_to_device(c, w.data(), (size_t)n * 4, nullptr, 0, false, &d_w, nullptr);
    if (rc) return rc;
    CU(cudaMemcpyAsync(sk.b_bs_w.as<float>() + sf.w_off, d_w, (size_t)n * 4, cudaMemcpyDeviceToDevice, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    return FYX_OK;
}

extern "C" int32_t fyx_reserve_skinning(fyx_ctx *c, uint64_t total_bones, uint64_t total_verts)
{
    if (!c) return FYX_ERR_INVALID_ARGUMENT;
    if (total_bones > 0xFFFFFFFFull) return fail(c, FYX_ERR_INVALID_ARGUMENT, "too many bones");
    CU(cudaSetDevice(c->device));
    // every surface is padded to a multiple of 4 vertices: leave room for 3 per surface (bounded by bones)
    return c->skin.grow(c, (uint32_t)total_bones, total_verts + 4 * total_bones + 4);
}

extern "C" int32_t fyx_commit_surfaces(fyx_ctx *c)
{
    if (!c) return FYX_ERR_INVALID_ARGUMENT;
    CU(cudaSetDevice(c->device));
    int32_t rc = c->skin.commit(c);
    if (rc) return rc;
    return sync_and_check(c);
}

// --------------------------------------------------------------------------------------------
// per frame.  Each stage is enqueued by one function that fyx_render_prep and the stage's own call share: scatter_locals,
// animate_enqueue (fyx_anim.inl), update_cull_enqueue, palette_enqueue, skin_enqueue.  They record no events; their callers do.
// --------------------------------------------------------------------------------------------
namespace {

// Hierarchy + world boxes, and the cull of the `nf` frusta prepare_cull set up (nf = 0: no cull).  With a LOD filter / static
// batches the cull cannot be fused into the level kernels: the pruning bits need every ancestor first.  side_fold_wanted: the
// caller joins c->ev_fold_done before the boxes are read, so the skinned-mesh fold may run on c->fold_stream (run_update);
// *side_fold tells whether it does.
int32_t update_cull_enqueue(fyx_ctx *c, uint32_t update_flags, uint32_t nf, bool side_fold_wanted = false, bool *side_fold = nullptr)
{
    static const bool side_fold_allowed = [] {
        const char *e = getenv("FYX_SIDE_FOLD"); // 0: the fold always runs in order on the main stream (A/B measurements)
        return !(e && *e == '0');
    }();
    const bool unf = unfused_cull(c, nf);
    const bool side = side_fold_wanted && side_fold_allowed && !unf && c->skin.n_fold;
    if (side_fold) *side_fold = side;
    int32_t rc = run_update(c, update_flags, (nf && !unf) ? &c->cp : nullptr, side ? c->fold_stream.h : nullptr);
    if (rc) return rc;
    return unf ? cull_unfused(c, nf) : FYX_OK;
}

// the bones' skinning matrices (palettes)
void palette_enqueue(fyx_ctx *c, cudaStream_t s)
{
    if (c->skin.n_entries) {
        launch_palette(s, c->a, c->skin.arrays());
        c->launches++;
    }
}

void skin_enqueue(fyx_ctx *c, cudaStream_t s)
{
    const Skinning &sk = c->skin;
    if (sk.n_tiles) {
        launch_skin(s, sk.arrays(), sk.b_tiles.as<SkinTile>(), sk.n_tiles, sk.max_bones, sk.any_blend_shapes);
        c->launches++;
    }
}

// A stand-alone stage call: the stage alone on the main stream, between EV_START and `ev_end`, synchronised; its time goes to `ms`.
template <class Enqueue> int32_t run_timed(fyx_ctx *c, int ev_end, float &ms, Enqueue enqueue)
{
    CU(cudaEventRecord(c->ev[EV_START], c->stream));
    int32_t rc = enqueue();
    if (rc) return rc;
    CU(cudaEventRecord(c->ev[ev_end], c->stream));
    rc = sync_and_check(c);
    cudaEventElapsedTime(&ms, c->ev[EV_START], c->ev[ev_end]);
    return rc;
}

} // namespace

extern "C" int32_t fyx_update_transforms(fyx_ctx *c, uint32_t update_flags)
{
    int32_t rc;
    if ((rc = enter(c)) || (rc = c->skin.commit(c))) return rc;
    return run_timed(c, EV_UPDATE, c->timings.update_ms, [&] { return update_cull_enqueue(c, update_flags, 0); });
}

// fyx_cull and fyx_update_and_cull prepare the cull even for nf = 0: a new, empty visible slot becomes the one fyx_get_visible reads
extern "C" int32_t fyx_cull(fyx_ctx *c, uint32_t nf, const fyx_frustum *fr, const uint32_t *cam_mask, const uint32_t *pass_flags)
{
    int32_t rc;
    if ((rc = enter(c)) || (rc = cull_prune_prepare(c, nf))) return rc;
    return run_timed(c, EV_CULL, c->timings.cull_ms, [&] {
        if ((rc = prepare_cull(c, nf, fr, cam_mask, pass_flags)) || !nf) return rc;
        return cull_unfused(c, nf);
    });
}

extern "C" int32_t fyx_update_and_cull(fyx_ctx *c, uint32_t update_flags, uint32_t nf, const fyx_frustum *fr,
                                       const uint32_t *cam_mask, const uint32_t *pass_flags)
{
    int32_t rc;
    if ((rc = enter(c)) || (rc = c->skin.commit(c)) || (rc = cull_prune_prepare(c, nf))) return rc;
    return run_timed(c, EV_UPDATE, c->timings.update_ms, [&] {
        return (rc = prepare_cull(c, nf, fr, cam_mask, pass_flags)) ? rc : update_cull_enqueue(c, update_flags, nf);
    });
}

extern "C" int32_t fyx_get_visible(fyx_ctx *c, uint32_t f, const uint32_t **out_idx, uint32_t *out_count)
{
    if (!c || !out_idx || !out_count) return FYX_ERR_INVALID_ARGUMENT;
    VisSlot &V = c->vs[c->readable];
    if (V.pending) return fail(c, FYX_ERR_STATE, "the frame is still in flight: call fyx_frame_wait first");
    if (f >= V.nf) return fail(c, FYX_ERR_INVALID_ARGUMENT, "frustum %u was not part of the last cull (%u frusta)", f, V.nf);
    CU(cudaSetDevice(c->device));
    int32_t rc = readback_visible(c, V, c->stream);
    if (rc) return rc;
    *out_idx = V.own_in_seg ? V.seg_own[f] : V.h_vis[f].as<uint32_t>(); // a gathered frame's own lists sit inside the node-wide host segment
    *out_count = V.h_counts.as<uint32_t>()[f];
    return FYX_OK;
}

extern "C" int32_t fyx_get_visible_device(fyx_ctx *c, uint32_t f, const uint32_t **d_idx, const uint32_t **d_count)
{
    if (!c || !d_idx || !d_count) return FYX_ERR_INVALID_ARGUMENT;
    VisSlot &V = c->vs[c->cur];
    if (f >= V.nf) return fail(c, FYX_ERR_INVALID_ARGUMENT, "frustum %u was not part of the last cull (%u frusta)", f, V.nf);
    *d_idx = V.b_vis[f].as<uint32_t>();
    *d_count = V.d_counts.as<uint32_t>() + f * kCountStride;
    return FYX_OK;
}

extern "C" int32_t fyx_build_palettes(fyx_ctx *c)
{
    int32_t rc;
    if ((rc = enter(c)) || (rc = c->skin.commit(c))) return rc;
    return run_timed(c, EV_PALETTE, c->timings.palette_ms, [&] {
        palette_enqueue(c, c->stream);
        return FYX_OK;
    });
}

extern "C" int32_t fyx_skin(fyx_ctx *c)
{
    int32_t rc;
    if ((rc = enter(c)) || (rc = c->skin.commit(c))) return rc;
    return run_timed(c, EV_SKIN, c->timings.skin_ms, [&] {
        skin_enqueue(c, c->stream);
        return FYX_OK;
    });
}

static void frame_timings_from_events(fyx_ctx *c)
{
    fyx_timings &t = c->timings;
    t.upload_ms = t.update_ms = t.palette_ms = t.skin_ms = t.readback_ms = 0.0f;
    if (c->stage_events_valid) {
        cudaEventElapsedTime(&t.upload_ms, c->ev[EV_START], c->ev[EV_UPLOAD]);
        cudaEventElapsedTime(&t.update_ms, c->ev[EV_UPLOAD], c->ev[EV_UPDATE]);
        cudaEventElapsedTime(&t.palette_ms, c->ev[EV_UPDATE], c->ev[EV_PALETTE]);
        cudaEventElapsedTime(&t.skin_ms, c->ev[EV_PALETTE], c->ev[EV_SKIN]);
        cudaEventElapsedTime(&t.readback_ms, c->ev[EV_SKIN], c->ev[EV_READBACK]);
    }
    cudaEventElapsedTime(&t.total_ms, c->ev[EV_START], c->ev[EV_READBACK]);
    t.cull_ms = 0.0f;
    c->timings_pending = false;
}

// 1. of fyx_render_prep: the changed local transforms.  Pinned caller memory is DMA'd in place (the caller keeps it untouched
//    until the frame is synchronised / waited for).  Async frames upload on the copy stream into alternating staging buffers,
//    so the H2D of frame i+1 overlaps the kernels of frame i.
static int32_t frame_upload(fyx_ctx *c, const fyx_frame_desc *fr, bool async)
{
    if (!fr->n_changed) return FYX_OK;
    const LocalsForm form = fr->changed_rot ? LOCALS_ROT : (fr->changed_trs ? LOCALS_TRS : LOCALS_M16);
    const void *payload = form == LOCALS_ROT ? static_cast<const void *>(fr->changed_rot)
                          : (form == LOCALS_TRS ? static_cast<const void *>(fr->changed_trs) : static_cast<const void *>(fr->changed_m16));
    if (!payload) return fail(c, FYX_ERR_INVALID_ARGUMENT, "changed_m16 / changed_trs / changed_rot is NULL");
    const size_t mb = (size_t)fr->n_changed * (form == LOCALS_ROT ? 16 : (form == LOCALS_TRS ? sizeof(fyx_trs) : 64)),
                 ib = fr->changed_idx ? (size_t)fr->n_changed * 4 : 0;
    cudaStream_t s = c->stream;
    int32_t rc;
    if (!(async && is_pinned(payload) && (!fr->changed_idx || is_pinned(fr->changed_idx)))) {
        void *d_m = nullptr, *d_i = nullptr;
        rc = stage_to_device(c, payload, mb, fr->changed_idx, ib, true, &d_m, &d_i);
        return rc ? rc : scatter_locals(c, s, form, fr->n_changed, static_cast<const uint32_t *>(d_i), d_m);
    }
    const int u = (c->upload_parity ^= 1);
    if (c->slot_used[u]) CU(cudaEventSynchronize(c->ev_slot_free[u])); // its previous scatter has consumed it
    const size_t off = (mb + 255) & ~size_t(255);
    rc = dev_ensure(c, c->d_stage_frame[u], off + ib + 256);
    if (rc) return rc;
    char *base = c->d_stage_frame[u].as<char>();
    const uint32_t *d_idx = ib ? reinterpret_cast<const uint32_t *>(base + off) : nullptr;
    CU(cudaMemcpyAsync(base, payload, mb, cudaMemcpyHostToDevice, c->copy_stream));
    if (ib) CU(cudaMemcpyAsync(base + off, fr->changed_idx, ib, cudaMemcpyHostToDevice, c->copy_stream));
    // The scatter writes local matrices / TRS records / F_DIRTY_SELF of the changed nodes — columns nothing of the PREVIOUS
    // frame reads once its level kernels and fold are done.  When that point is known (the previous frame recorded its
    // cull event) and nothing else has been enqueued on the main stream since, the scatter runs on the copy stream, beside
    // the previous frame's palette / skinning kernels, instead of in front of this frame's level kernels.  Nor may the
    // scatter enqueue anything on the main stream itself: a TRS form's first upload fills the TRS column there.
    static const bool side_allowed = [] {
        const char *e = getenv("FYX_SIDE_SCATTER"); // 0: always scatter on the main stream (A/B measurements)
        return !(e && *e == '0');
    }();
    const bool side = side_allowed && c->ev_levels_prev && c->launches == c->launches_at_frame_end &&
                      (form == LOCALS_M16 || c->trs.live) && !(fr->struct_size >= sizeof(fyx_frame_desc) && fr->do_animate);
    if (side) {
        CU(cudaStreamWaitEvent(c->copy_stream, c->ev_levels_prev, 0));
        if ((rc = scatter_locals(c, c->copy_stream, form, fr->n_changed, d_idx, base))) return rc;
        CU(cudaEventRecord(c->ev_upload[u], c->copy_stream));
        CU(cudaEventRecord(c->ev_slot_free[u], c->copy_stream));
        CU(cudaStreamWaitEvent(s, c->ev_upload[u], 0));
    } else {
        CU(cudaEventRecord(c->ev_upload[u], c->copy_stream));
        CU(cudaStreamWaitEvent(s, c->ev_upload[u], 0));
        if ((rc = scatter_locals(c, s, form, fr->n_changed, d_idx, base))) return rc;
        CU(cudaEventRecord(c->ev_slot_free[u], s));
    }
    c->slot_used[u] = true;
    return FYX_OK;
}

extern "C" int32_t fyx_render_prep(fyx_ctx *c, const fyx_frame_desc *fr)
{
    if (!c || !fr) return FYX_ERR_INVALID_ARGUMENT;
    if (fr->struct_size < offsetof(fyx_frame_desc, do_animate)) return fail(c, FYX_ERR_INVALID_ARGUMENT, "fyx_frame_desc.struct_size too small");
    int32_t rc;
    if ((rc = enter(c)) || (rc = c->skin.commit(c)) || (rc = cull_prune_prepare(c, fr->n_frusta))) return rc;
    cudaStream_t s = c->stream;
    CU(cudaEventRecord(c->ev[EV_START], s));
    // 0. animation players tick before Graph::update (N2): curves are device-resident, nothing to upload
    if (fr->struct_size >= sizeof(fyx_frame_desc) && fr->do_animate) {
        rc = animate_enqueue(c, fr->animate_dt);
        if (rc) return rc;
    }
    const bool async = (fr->flags & FYX_FRAME_ASYNC) != 0;
    // Per-stage events sit BETWEEN kernels of the programmatic-dependent-launch chain and would keep a kernel's
    // prologue from overlapping its predecessor's tail: only synchronous frames record them (their timings are read
    // right after the call); asynchronous frames record the frame's start and end only (stage fields read 0).
    const bool stage_events = !async;
    c->stage_events_valid = stage_events;
    const bool pipelined = async && fr->readback_visible && fr->n_frusta; // read-back deferred to fyx_frame_wait
    // 1. changed local transforms
    if ((rc = frame_upload(c, fr, async))) return rc;
    if (stage_events) CU(cudaEventRecord(c->ev[EV_UPLOAD], s));
    // 2. hierarchy + world boxes + cull; an asynchronous frame that goes on to skinning joins a fold on the side below
    if (fr->n_frusta) {
        rc = prepare_cull(c, fr->n_frusta, fr->frusta, fr->cam_mask, fr->pass_flags);
        if (rc) return rc;
    }
    bool side_fold = false;
    if ((rc = update_cull_enqueue(c, fr->update_flags, fr->n_frusta, async && fr->do_skin && c->skin.n_tiles, &side_fold))) return rc;
    if (stage_events) CU(cudaEventRecord(c->ev[EV_UPDATE], s));
    c->ev_levels_prev = nullptr;
    if (fr->n_frusta && (async || (fr->flags & FYX_FRAME_ALLGATHER))) {
        // consumed by the read-back / collective streams and by the next frame's scatter: the lists are complete after the fold
        CU(cudaEventRecord(c->vs[c->cur].ev_cull, side_fold ? c->fold_stream : s));
        c->ev_levels_prev = c->vs[c->cur].ev_cull;
    }
    // multi-GPU: the visible lists are complete here; their all-gather runs on the collective stream beside
    // the palette / skinning kernels below (the path's one exchange step, SURVEY §8e)
    const bool gather = (fr->flags & FYX_FRAME_ALLGATHER) && fr->n_frusta;
    if (gather) {
        if (!c->comm) return fail(c, FYX_ERR_STATE, "FYX_FRAME_ALLGATHER without fyx_comm_init");
        CU(cudaStreamWaitEvent(c->comm_stream, c->vs[c->cur].ev_cull, 0));
        if (c->vs[c->cur ^ 1].gathered) CU(cudaStreamWaitEvent(c->comm_stream, c->vs[c->cur ^ 1].ev_gather, 0)); // a stand-alone exchange of the previous frame
        c->vs[c->cur].host_copy_private = !fr->readback_visible; // nobody promised that every rank fetches this frame's lists
        rc = allgather_enqueue(c, c->vs[c->cur], c->comm_stream);
        if (rc) return rc;
    }
    // 3. palettes, 4. skinning
    if (fr->do_palettes) palette_enqueue(c, s);
    if (stage_events) CU(cudaEventRecord(c->ev[EV_PALETTE], s));
    if (fr->do_skin) skin_enqueue(c, s);
    if (stage_events) CU(cudaEventRecord(c->ev[EV_SKIN], s));
    CU(cudaGetLastError());
    if (side_fold) CU(cudaStreamWaitEvent(s, c->ev_fold_done, 0)); // join: whatever follows on the main stream sees the folded boxes and the complete lists
    if (gather) {
        // the host waits only for the cull + the counts (the skinning kernel keeps running), then enqueues the payload
        rc = allgather_finish(c, c->vs[c->cur], c->comm_stream);
        if (rc) return rc;
        CU(cudaEventRecord(c->ev_x1[c->vs[c->cur].epoch & 1], c->comm_stream));
        CU(cudaEventRecord(c->vs[c->cur].ev_gather, c->comm_stream));
        CU(cudaStreamWaitEvent(s, c->vs[c->cur].ev_gather, 0)); // the frame is complete when the gathered lists are
    }
    // 5. visible lists to the host
    VisSlot &V = c->vs[c->cur];
    if (pipelined) {
        // deferred: counts travel on the read-back stream as soon as the cull is done; fyx_frame_wait fetches the lists
        CU(cudaEventRecord(V.ev_done, s));
        CU(cudaStreamWaitEvent(c->d2h_stream, V.ev_cull, 0));
        CU(cudaMemcpy2DAsync(V.h_counts.p, sizeof(uint32_t), V.d_counts.p, sizeof(uint32_t) * kCountStride, sizeof(uint32_t), V.nf,
                             cudaMemcpyDeviceToHost, c->d2h_stream));
        CU(cudaEventRecord(V.ev_counts, c->d2h_stream));
        V.pending = true;
        V.own_only = gather && (fr->flags & FYX_FRAME_READBACK_OWN);
        V.frame_no = ++c->frame_counter;
    } else if (fr->readback_visible && fr->n_frusta && !gather) {
        rc = readback_visible(c, V, s);
        if (rc) return rc;
    } // with FYX_FRAME_ALLGATHER the frame's result is the gathered lists: fyx_get_visible_gathered fetches them
    CU(cudaEventRecord(c->ev[EV_READBACK], s));
    c->launches_at_frame_end = c->launches;
    if (async) {
        c->timings_pending = true;
        return FYX_OK;
    }
    rc = sync_and_check(c);
    frame_timings_from_events(c);
    if (!rc && gather && fr->readback_visible && c->hostseg_ready) rc = hostseg_publish(c, V, s); // every rank's part, without being asked
    return rc;
}

// Collect the oldest pipelined frame: wait for its kernels, bring its visible lists to the host, make it
// the frame fyx_get_visible reads.  No-op when nothing is in flight.
extern "C" int32_t fyx_frame_wait(fyx_ctx *c)
{
    if (!c) return FYX_ERR_INVALID_ARGUMENT;
    int slot = -1;
    for (int i = 0; i < 2; ++i)
        if (c->vs[i].pending && (slot < 0 || c->vs[i].frame_no < c->vs[slot].frame_no)) slot = i;
    if (slot < 0) return FYX_OK;
    CU(cudaSetDevice(c->device));
    VisSlot &V = c->vs[slot];
    CU(cudaEventSynchronize(V.ev_counts));
    V.counts_on_host = true;
    const bool seg = V.gathered && c->hostseg_ready && !V.host_copy_private;
    const bool own = !seg && (!V.gathered || V.own_only);
    for (uint32_t f = 0; f < V.nf && own; ++f) {
        const size_t n = V.h_counts.as<uint32_t>()[f];
        CU(V.h_vis[f].ensure(n * sizeof(uint32_t)));
        if (n) CU(cudaMemcpyAsync(V.h_vis[f].p, V.b_vis[f].p, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, c->d2h_stream));
    }
    if (seg) {
        // multi-GPU frame: this rank's own lists go into the node-wide host segment at their offsets (every rank does the
        // same over its own PCIe link); fyx_get_visible_gathered reads the whole lists there
        int32_t rc = hostseg_publish(c, V, c->d2h_stream);
        if (rc) return rc;
    } else if (V.gathered && !V.own_only) { // no segment: the host wants the whole (all-gathered) lists from this rank's device
        int32_t rc = resolve_counts(c, V);
        if (rc) return rc;
        CU(cudaStreamWaitEvent(c->d2h_stream, V.ev_gather, 0));
        for (uint32_t f = 0; f < V.nf; ++f) {
            const size_t n = V.gath_count[f];
            CU(V.h_gath[f].ensure(n * sizeof(uint32_t)));
            if (n) CU(cudaMemcpyAsync(V.h_gath[f].p, V.gath_ptr[f], n * sizeof(uint32_t), cudaMemcpyDeviceToHost, c->d2h_stream));
        }
        CU(cudaEventRecord(c->ev_gath_read[V.epoch & 1], c->d2h_stream));
        c->gath_read_valid[V.epoch & 1] = true;
        V.gathered_on_host = true;
    }
    CU(cudaStreamWaitEvent(c->d2h_stream, V.ev_done, 0)); // the error word is final once the frame's last kernel ran
    CU(cudaMemcpyAsync(c->h_err.p, c->d_err.p, sizeof(uint32_t), cudaMemcpyDeviceToHost, c->d2h_stream));
    CU(cudaStreamSynchronize(c->d2h_stream));
    V.lists_on_host = own || V.own_in_seg;
    V.pending = false;
    c->readable = slot;
    return check_device_errors(c);
}

// --------------------------------------------------------------------------------------------
// read-back
// --------------------------------------------------------------------------------------------
namespace {
// gather `count` items of `item_bytes` through a gather launcher into caller memory
template <class Launch> int32_t gather_out(fyx_ctx *c, uint32_t count, const uint32_t *idx, size_t item_bytes, void *out, Launch launch)
{
    if (int32_t rc = topology_check(c)) return rc;
    if (!count) return FYX_OK;
    if (!out) return fail(c, FYX_ERR_INVALID_ARGUMENT, "output pointer is NULL");
    CU(cudaSetDevice(c->device));
    const size_t out_bytes = (size_t)count * item_bytes;
    const size_t idx_bytes = idx ? (((size_t)count * 4 + 255) & ~size_t(255)) : 0;
    int32_t rc = dev_ensure(c, c->d_stage, idx_bytes + out_bytes);
    if (rc) return rc;
    char *base = c->d_stage.as<char>();
    uint32_t *d_idx = nullptr;
    if (idx) {
        CU(cudaStreamSynchronize(c->stream));
        CU(cudaMemcpyAsync(base, idx, (size_t)count * 4, cudaMemcpyHostToDevice, c->stream));
        d_idx = reinterpret_cast<uint32_t *>(base);
    }
    launch(d_idx, base + idx_bytes);
    c->launches++;
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(out, base + idx_bytes, out_bytes, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    return FYX_OK;
}
} // namespace

extern "C" int32_t fyx_get_global_matrices(fyx_ctx *c, uint32_t count, const uint32_t *idx, float *out)
{
    return gather_out(c, count, idx, 64, out, [&](uint32_t *d_idx, void *d_out) {
        launch_gather_globals(c->stream, c->a, count, d_idx, c->b_slot_of_node.as<uint32_t>(), c->n_nodes, static_cast<float *>(d_out));
    });
}

extern "C" int32_t fyx_get_world_aabbs(fyx_ctx *c, uint32_t count, const uint32_t *idx, float *out)
{
    return gather_out(c, count, idx, 24, out, [&](uint32_t *d_idx, void *d_out) {
        launch_gather_aabbs(c->stream, c->a, count, d_idx, c->b_slot_of_node.as<uint32_t>(), c->n_nodes, static_cast<float *>(d_out));
    });
}

extern "C" int32_t fyx_get_global_flags(fyx_ctx *c, uint32_t count, const uint32_t *idx, uint32_t *out)
{
    return gather_out(c, count, idx, 4, out, [&](uint32_t *d_idx, void *d_out) {
        launch_gather_flags(c->stream, c->a, count, d_idx, c->b_slot_of_node.as<uint32_t>(), c->n_nodes, static_cast<uint32_t *>(d_out));
    });
}

extern "C" int32_t fyx_get_palette(fyx_ctx *c, uint32_t sid, float *out)
{
    if (!c || !out) return FYX_ERR_INVALID_ARGUMENT;
    if (sid >= c->skin.surfaces.size()) return fail(c, FYX_ERR_INVALID_ARGUMENT, "surface id %u out of range", sid);
    CU(cudaSetDevice(c->device));
    const SkinSurface &sf = c->skin.surfaces[sid];
    if (!sf.n_bones()) return FYX_OK;
    CU(cudaMemcpyAsync(out, c->skin.b_palette.as<float>() + 16 * (size_t)sf.bone_off, (size_t)sf.n_bones() * 64, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    return FYX_OK;
}

extern "C" int32_t fyx_get_skinned(fyx_ctx *c, uint32_t sid, float *out_pos, float *out_nrm)
{
    if (!c) return FYX_ERR_INVALID_ARGUMENT;
    if (sid >= c->skin.surfaces.size()) return fail(c, FYX_ERR_INVALID_ARGUMENT, "surface id %u out of range", sid);
    CU(cudaSetDevice(c->device));
    const SkinSurface &sf = c->skin.surfaces[sid];
    if (!sf.n_verts) return FYX_OK;
    if (out_pos) CU(cudaMemcpyAsync(out_pos, c->skin.b_opos.as<float>() + 3 * sf.vert_off, (size_t)sf.n_verts * 12, cudaMemcpyDeviceToHost, c->stream));
    if (out_nrm) CU(cudaMemcpyAsync(out_nrm, c->skin.b_onrm.as<float>() + 3 * sf.vert_off, (size_t)sf.n_verts * 12, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    return FYX_OK;
}

extern "C" int32_t fyx_get_skinned_device(fyx_ctx *c, uint32_t sid, const float **d_pos, const float **d_nrm)
{
    if (!c) return FYX_ERR_INVALID_ARGUMENT;
    if (sid >= c->skin.surfaces.size()) return fail(c, FYX_ERR_INVALID_ARGUMENT, "surface id %u out of range", sid);
    const SkinSurface &sf = c->skin.surfaces[sid];
    if (d_pos) *d_pos = c->skin.b_opos.as<float>() + 3 * sf.vert_off;
    if (d_nrm) *d_nrm = c->skin.b_onrm.as<float>() + 3 * sf.vert_off;
    return FYX_OK;
}

extern "C" int32_t fyx_get_timings(fyx_ctx *c, fyx_timings *out)
{
    if (!c || !out) return FYX_ERR_INVALID_ARGUMENT;
    if (c->timings_pending) {
        CU(cudaSetDevice(c->device));
        CU(cudaEventSynchronize(c->ev[EV_READBACK]));
        frame_timings_from_events(c);
    }
    *out = c->timings;
    return FYX_OK;
}

#include "fyx_comm.inl"
#include "fyx_drawprep.inl"
#include "fyx_anim.inl"
