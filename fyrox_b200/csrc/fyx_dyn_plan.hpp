// fyx_dyn_plan.hpp — dynamic batching's host rules: the registrations of Dynamic meshes (fyx_add_dynamic_surface) and the quad
// nodes (fyx_set_sprites) with the layout ids and batch keys they share, the checks of both calls, the pools' compaction, the
// device tables in push order and the placement of a pack's segments.  Host code only, with no CUDA types, so that the CPU
// tests build it with g++ alone.
#pragma once
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <set>
#include <unordered_map>
#include <unordered_set>
#include <utility>
#include <vector>

#include "../../include/fyrox_b200.h"
#include "fyx_slots.hpp"

namespace fyx {

// Dynamic batching (scene/mesh/mod.rs:739-753, 804-833; renderer/bundle.rs:1177-1243).  The registered surfaces and the quad
// nodes (fyx_set_sprites: one item of 4 vertices and 2 triangles each), in the reference's push order: dynamic nodes ordered by
// DFS rank (else node index), each node's surfaces by ordinal.
constexpr uint32_t kDynMesh = 0u; // DynItemDev::kind of a registered surface; else FYX_SPRITE_3D / FYX_SPRITE_RECTANGLE
struct DynItemDev {
    uint32_t node, slot, batch_key, layout;
    uint32_t n_verts, n_tris;
    uint32_t tri_src;   // first u32 of its triangles in the registration pool
    uint32_t kind;
    uint64_t vtx_src;   // first byte of its vertices in the registration pool (16-byte aligned)
};
struct DynLayoutDev {
    uint32_t stride, pos, nrm, tan; // attribute offsets, FYX_NONE = not transformed
};
static_assert(sizeof(DynItemDev) == 40 && sizeof(DynLayoutDev) == 16, "the records the k_dyn_* kernels read");

constexpr uint64_t kDynTriPool = 1ull << 32; // a registration's triangles end below this word of the pool: tri_src is a u32

// One registered surface (fyx_add_dynamic_surface) and one quad node (fyx_set_sprites; kind 0 = not a quad node)
struct DynReg {
    uint32_t id, node, ordinal, batch_key, layout, n_verts, n_tris, tri_src;
    uint64_t vtx_src;
};
struct DynQuad {
    uint32_t kind, batch_key, layout_id;
};

// Surface `ordinal` of a node as fyx_set_node_surfaces left it; only a batchable one is batched
enum class DynSurface { kMissing, kSkinned, kBatchable };

// One call's claims of layout ids (with their layouts) and batch keys (with their layout ids), staged until the call succeeds
struct DynClaims {
    std::unordered_map<uint32_t, fyx_dynamic_layout> layout;
    std::unordered_map<uint32_t, uint32_t> key;
};

// The checks below refuse a call by returning fail(FYX_ERR_* code, printf format, arguments...); they return FYX_OK otherwise,
// and a refused call changes nothing.  surface(node, ordinal) answers DynSurface.
struct DynRegistry {
    std::vector<DynReg> regs;
    std::set<uint64_t> pairs; // node << 32 | ordinal of every registration
    NodeRecords<DynQuad> quad_of_node{DynQuad{0u, 0u, 0u}};
    std::vector<uint32_t> quad_seen; // by node index: the fyx_set_sprites call that last listed it (duplicate check)
    uint32_t quad_call = 0;
    std::vector<fyx_dynamic_layout> layouts; // by layout id; stride FYX_NONE = nothing uses it
    std::vector<uint32_t> key_layout;        // by batch key; FYX_NONE = nothing uses it
    uint64_t vtx_used = 0, tri_used = 0;     // pools: vertex bytes (each surface 16-byte aligned), triangle words
    uint32_t next_id = 0;

    template <class Fail> static int32_t check_alive(uint32_t node, const std::vector<uint32_t> &slot_of_node, Fail fail)
    {
        if (node >= slot_of_node.size() || slot_of_node[node] == FYX_NONE) return fail(FYX_ERR_INVALID_ARGUMENT, "node %u is not alive", node);
        return FYX_OK;
    }
    template <class Fail> static int32_t check_ids(uint32_t batch_key, uint32_t layout_id, Fail fail)
    {
        if (batch_key >= (1u << 24)) return fail(FYX_ERR_INVALID_ARGUMENT, "batch key %u too large: keys must be dense (< 2^24)", batch_key);
        if (layout_id >= (1u << 16)) return fail(FYX_ERR_INVALID_ARGUMENT, "layout id %u too large: ids must be dense (< 2^16)", layout_id);
        return FYX_OK;
    }
    bool registered(uint32_t node) const
    {
        const auto it = pairs.lower_bound((uint64_t)node << 32);
        return it != pairs.end() && (*it >> 32) == node;
    }
    // a claim of `layout_id` for `ly` and of `batch_key` for `layout_id`: refused when the committed tables or `staged` give
    // either to another, else added to `staged`
    template <class Fail> int32_t claim(uint32_t layout_id, const fyx_dynamic_layout &ly, uint32_t batch_key, DynClaims &staged, Fail fail) const
    {
        fyx_dynamic_layout given = layout_id < layouts.size() ? layouts[layout_id] : fyx_dynamic_layout{FYX_NONE, FYX_NONE, FYX_NONE, FYX_NONE};
        uint32_t key_id = batch_key < key_layout.size() ? key_layout[batch_key] : FYX_NONE;
        if (auto it = staged.layout.find(layout_id); it != staged.layout.end()) given = it->second;
        if (auto it = staged.key.find(batch_key); it != staged.key.end()) key_id = it->second;
        if (given.stride != FYX_NONE && memcmp(&given, &ly, sizeof ly) != 0)
            return fail(FYX_ERR_INVALID_ARGUMENT, "layout id %u was given with another layout", layout_id);
        if (key_id != FYX_NONE && key_id != layout_id)
            return fail(FYX_ERR_INVALID_ARGUMENT, "batch key %u was given with layout %u: one bundle holds one vertex layout", batch_key, key_id);
        staged.layout[layout_id] = ly;
        staged.key[batch_key] = layout_id;
        return FYX_OK;
    }

    // fyx_add_dynamic_surface's checks; the layout id and batch key are claimed in `claims`
    template <class Surface, class Fail>
    int32_t check_surface(uint32_t node, uint32_t ordinal, uint32_t batch_key, uint32_t layout_id, const fyx_dynamic_layout *layout,
                          uint32_t n_verts, const void *verts, uint32_t n_tris, const uint32_t *tris,
                          const std::vector<uint32_t> &slot_of_node, Surface surface, DynClaims &claims, Fail fail) const
    {
        if (!layout || (n_verts && !verts) || (n_tris && !tris)) return fail(FYX_ERR_INVALID_ARGUMENT, "layout / verts / triangles is NULL");
        if (int32_t rc = check_alive(node, slot_of_node, fail)) return rc;
        if (n_verts >= 256) return fail(FYX_ERR_INVALID_ARGUMENT, "%u vertices: only surfaces of fewer than 256 vertices are batched", n_verts);
        if (int32_t rc = check_ids(batch_key, layout_id, fail)) return rc;
        const fyx_dynamic_layout &ly = *layout;
        if (!ly.stride) return fail(FYX_ERR_INVALID_ARGUMENT, "the layout's stride is 0");
        const uint32_t sizes[3] = {12u, 12u, 16u}, offs[3] = {ly.position_offset, ly.normal_offset, ly.tangent_offset};
        for (int k = 0; k < 3; ++k)
            if (offs[k] != FYX_NONE && (uint64_t)offs[k] + sizes[k] > ly.stride)
                return fail(FYX_ERR_INVALID_ARGUMENT, "attribute at offset %u does not fit the stride %u", offs[k], ly.stride);
        const DynSurface sf = surface(node, ordinal);
        if (sf == DynSurface::kMissing) return fail(FYX_ERR_INVALID_ARGUMENT, "node %u has no surface %u", node, ordinal);
        if (sf == DynSurface::kSkinned) return fail(FYX_ERR_INVALID_ARGUMENT, "surface %u of node %u is skinned: it is pushed, not batched", ordinal, node);
        if (pairs.count((uint64_t)node << 32 | ordinal))
            return fail(FYX_ERR_INVALID_ARGUMENT, "surface %u of node %u is already registered", ordinal, node);
        if (quad_of_node[node].kind)
            return fail(FYX_ERR_INVALID_ARGUMENT, "node %u is a sprite or rectangle (fyx_set_sprites): it has no mesh surfaces", node);
        if (int32_t rc = claim(layout_id, ly, batch_key, claims, fail)) return rc;
        for (uint64_t k = 0; k < (uint64_t)n_tris * 3; ++k)
            if (tris[k] >= n_verts) return fail(FYX_ERR_INVALID_ARGUMENT, "triangle index %u out of range (%u vertices)", tris[k], n_verts);
        if (tri_used + (uint64_t)n_tris * 3 >= kDynTriPool)
            return fail(FYX_ERR_INVALID_ARGUMENT, "%u triangles do not fit the triangle pool (%llu of its 2^32 words in use)", n_tris,
                        (unsigned long long)tri_used);
        return FYX_OK;
    }
    // A checked surface whose data now sits at the pools' ends (vtx_used, tri_used): its id
    uint32_t add_surface(uint32_t node, uint32_t ordinal, uint32_t batch_key, uint32_t layout_id, uint32_t n_verts, uint32_t n_tris,
                         const DynClaims &claims)
    {
        commit(claims);
        regs.push_back(DynReg{next_id, node, ordinal, batch_key, layout_id, n_verts, n_tris, (uint32_t)tri_used, vtx_used});
        pairs.insert((uint64_t)node << 32 | ordinal);
        vtx_used = (vtx_used + (uint64_t)n_verts * layouts[layout_id].stride + 15) & ~uint64_t(15);
        tri_used += (uint64_t)n_tris * 3;
        return next_id++;
    }

    // fyx_set_sprites's checks of a non-empty call whose records are present; the ids and keys of changed records are claimed
    // in `claims`.  has_surfaces(node) / skinned(node): fyx_set_node_surfaces gave the node surfaces / it has a skinned surface.
    template <class HasSurfaces, class Skinned, class Fail>
    int32_t check_sprites(uint32_t count, const uint32_t *idx, const fyx_sprite *rec, const std::vector<uint32_t> &slot_of_node,
                          HasSurfaces has_surfaces, Skinned skinned, DynClaims &claims, Fail fail)
    {
        // a node listed twice: the per-node stamp of this call (no allocation per record; an appearance update of many records
        // is the common call)
        if (quad_seen.size() < slot_of_node.size()) quad_seen.resize(slot_of_node.size(), 0u);
        if (++quad_call == 0u) {
            std::fill(quad_seen.begin(), quad_seen.end(), 0u);
            quad_call = 1u;
        }
        for (uint32_t k = 0; k < count; ++k) {
            const uint32_t node = idx ? idx[k] : k;
            const fyx_sprite &r = rec[k];
            if (r.kind != FYX_SPRITE_3D && r.kind != FYX_SPRITE_RECTANGLE) return fail(FYX_ERR_INVALID_ARGUMENT, "record %u: unknown kind %u", k, r.kind);
            if (int32_t rc = check_alive(node, slot_of_node, fail)) return rc;
            if (quad_seen[node] == quad_call) return fail(FYX_ERR_INVALID_ARGUMENT, "node %u is listed twice", node);
            quad_seen[node] = quad_call;
            if (int32_t rc = check_ids(r.batch_key, r.layout_id, fail)) return rc;
            const DynQuad old = quad_of_node[node];
            if (old.kind == r.kind && old.batch_key == r.batch_key && old.layout_id == r.layout_id) continue; // the records alone change
            if (!old.kind) { // a new quad node
                if (has_surfaces(node)) return fail(FYX_ERR_INVALID_ARGUMENT, "node %u has mesh surfaces (fyx_set_node_surfaces)", node);
                if (skinned(node)) return fail(FYX_ERR_INVALID_ARGUMENT, "node %u has a skinned surface", node);
                if (registered(node)) return fail(FYX_ERR_INVALID_ARGUMENT, "node %u has dynamic-surface registrations", node);
            }
            const fyx_dynamic_layout quad_layout{r.kind == FYX_SPRITE_3D ? 40u : 24u, 0u, FYX_NONE, FYX_NONE};
            if (int32_t rc = claim(r.layout_id, quad_layout, r.batch_key, claims, fail)) return rc;
        }
        return FYX_OK;
    }
    // The checked records of fyx_set_sprites: false when no kind, batch key or layout id changed (the tables stay)
    bool set_sprites(uint32_t count, const uint32_t *idx, const fyx_sprite *rec, const DynClaims &claims)
    {
        if (claims.key.empty()) return false;
        for (uint32_t k = 0; k < count; ++k) quad_of_node.set(idx ? idx[k] : k, DynQuad{rec[k].kind, rec[k].batch_key, rec[k].layout_id});
        commit(claims);
        release(); // frees what the changed nodes no longer use
        return true;
    }

    // fyx_clear_dynamic_surfaces / fyx_clear_sprites of the listed nodes (nodes NULL = every node)
    void clear_surfaces(uint32_t count, const uint32_t *nodes)
    {
        const std::unordered_set<uint32_t> drop(nodes, nodes ? nodes + count : nodes);
        regs.erase(std::remove_if(regs.begin(), regs.end(), [&](const DynReg &r) { return !nodes || drop.count(r.node); }), regs.end());
        release();
    }
    void clear_sprites(uint32_t count, const uint32_t *nodes)
    {
        if (!nodes) quad_of_node.rec.clear();
        else
            for (uint32_t k = 0; k < count; ++k)
                if (nodes[k] < quad_of_node.rec.size()) quad_of_node.rec[nodes[k]] = quad_of_node.def;
        release();
    }
    // a node that is not alive any more drops its registrations and its quad record
    void topology_changed(const std::vector<uint32_t> &old_slot_of_node, const std::vector<uint32_t> &new_slot_of_node)
    {
        quad_of_node.topology_changed(old_slot_of_node, new_slot_of_node);
        regs.erase(std::remove_if(regs.begin(), regs.end(),
                                  [&](const DynReg &r) { return r.node >= new_slot_of_node.size() || new_slot_of_node[r.node] == FYX_NONE; }),
                   regs.end());
        release();
    }

    void commit(const DynClaims &staged)
    {
        for (const auto &[id, ly] : staged.layout) {
            if (layouts.size() <= id) layouts.resize(id + 1, fyx_dynamic_layout{FYX_NONE, FYX_NONE, FYX_NONE, FYX_NONE});
            layouts[id] = ly;
        }
        for (const auto &[key, id] : staged.key) {
            if (key_layout.size() <= key) key_layout.resize(key + 1, FYX_NONE);
            key_layout[key] = id;
        }
    }
    // after registrations or quad nodes went: their pairs, and the layout ids and batch keys nothing uses, go
    void release()
    {
        pairs.clear();
        std::vector<uint8_t> key_used(key_layout.size(), 0), layout_used(layouts.size(), 0);
        for (const DynReg &r : regs) {
            pairs.insert((uint64_t)r.node << 32 | r.ordinal);
            key_used[r.batch_key] = layout_used[r.layout] = 1;
        }
        for (const DynQuad &q : quad_of_node.rec)
            if (q.kind) key_used[q.batch_key] = layout_used[q.layout_id] = 1;
        for (size_t k = 0; k < key_used.size(); ++k)
            if (!key_used[k]) key_layout[k] = FYX_NONE;
        for (size_t l = 0; l < layout_used.size(); ++l)
            if (!layout_used[l]) layouts[l].stride = FYX_NONE;
    }
};

// The pools keep a registration's bytes until the flush after it is dropped: once more than half of either pool is dropped
// registrations, the live ones move to fresh pools, in registration order, each one's vertices 16-byte aligned.
struct DynCompaction {
    bool compact = false;
    std::vector<DynReg> regs;          // the registrations at their offsets in the fresh pools
    uint64_t vtx_used = 0, tri_used = 0; // of the fresh pools
};
inline DynCompaction plan_dyn_compaction(const DynRegistry &r)
{
    DynCompaction p;
    uint64_t live_v = 0, live_t = 0;
    for (const DynReg &g : r.regs) {
        live_v += ((uint64_t)g.n_verts * r.layouts[g.layout].stride + 15) & ~uint64_t(15);
        live_t += (uint64_t)g.n_tris * 3;
    }
    p.compact = 2 * live_v < r.vtx_used || 2 * live_t < r.tri_used;
    if (!p.compact) return p;
    p.regs = r.regs;
    for (DynReg &g : p.regs) {
        g.vtx_src = p.vtx_used;
        g.tri_src = (uint32_t)p.tri_used;
        p.vtx_used += ((uint64_t)g.n_verts * r.layouts[g.layout].stride + 15) & ~uint64_t(15);
        p.tri_used += (uint64_t)g.n_tris * 3;
    }
    return p;
}

// The device tables in push order: of_slot (per slot: the node's dense dynamic index, FYX_NONE = none), item_first (per
// dynamic node, then the end), per item its ordinal (FYX_NONE for a quad node: every surface of the node is left out of the
// instances) and record, and the device layouts of layout ids 0 .. the largest an item uses.
struct DynItemPlan {
    std::vector<uint32_t> of_slot, item_first, ordinal;
    std::vector<DynItemDev> items;
    std::vector<DynLayoutDev> layouts;
    uint32_t n_quads = 0;
};
// dfs_rank: the node's rank in the reference's DFS, nullptr = node index order.  A registered surface that surface() does not
// call batchable (removed or named skinned since) is pushed, not batched.
template <class Surface>
DynItemPlan plan_dyn_items(const DynRegistry &r, const std::vector<uint32_t> &slot_of_node, uint32_t n_slots, const uint32_t *dfs_rank, Surface surface)
{
    std::vector<std::pair<uint32_t, DynItemDev>> order; // (ordinal, item)
    for (const DynReg &g : r.regs)
        if (surface(g.node, g.ordinal) == DynSurface::kBatchable)
            order.push_back({g.ordinal, DynItemDev{g.node, slot_of_node[g.node], g.batch_key, g.layout, g.n_verts, g.n_tris, g.tri_src, kDynMesh, g.vtx_src}});
    for (uint32_t n = 0; n < (uint32_t)r.quad_of_node.rec.size(); ++n) {
        const DynQuad q = r.quad_of_node.rec[n];
        if (q.kind) order.push_back({FYX_NONE, DynItemDev{n, slot_of_node[n], q.batch_key, q.layout_id, 4u, 2u, 0u, q.kind, 0u}});
    }
    auto rank = [&](uint32_t n) { return dfs_rank ? dfs_rank[n] : n; };
    std::sort(order.begin(), order.end(), [&](const auto &x, const auto &y) {
        const uint32_t rx = rank(x.second.node), ry = rank(y.second.node);
        return rx != ry ? rx < ry : (x.second.node != y.second.node ? x.second.node < y.second.node : x.first < y.first);
    });
    DynItemPlan p;
    p.of_slot.assign(std::max<uint32_t>(n_slots, 1), FYX_NONE);
    uint32_t n_layouts = 0;
    for (size_t k = 0; k < order.size(); ++k) {
        const DynItemDev &it = order[k].second;
        if (k == 0 || order[k - 1].second.node != it.node) {
            p.of_slot[it.slot] = (uint32_t)p.item_first.size();
            p.item_first.push_back((uint32_t)p.items.size());
        }
        p.items.push_back(it);
        p.ordinal.push_back(order[k].first);
        n_layouts = std::max(n_layouts, it.layout + 1);
        p.n_quads += it.kind != kDynMesh ? 1u : 0u;
    }
    p.item_first.push_back((uint32_t)p.items.size());
    p.layouts.assign(n_layouts, DynLayoutDev{1u, FYX_NONE, FYX_NONE, FYX_NONE});
    for (uint32_t l = 0; l < n_layouts && l < r.layouts.size(); ++l) {
        const fyx_dynamic_layout &ly = r.layouts[l];
        if (ly.stride != FYX_NONE) p.layouts[l] = DynLayoutDev{ly.stride, ly.position_offset, ly.normal_offset, ly.tangent_offset};
    }
    return p;
}

// Where a pack's dynamic pass puts every segment's items, hash tables and (segment, layout) streams
struct DynPlacement {
    std::vector<uint32_t> item0, stream0; // [segments + 1]: first item, first stream of each segment, then the ends
    std::vector<uint32_t> hash0, hmask;   // [segments]: first entry of the segment's two hash tables, entries per table - 1
    std::vector<uint32_t> stream_tri;     // [segments * layouts]: first output triangle of each (segment, layout) stream
    std::vector<uint64_t> stream_vtx;     // [segments * layouts]: its first output byte (16-byte aligned)
    std::vector<fyx_dynamic_stream> streams; // per segment one per layout with items, ascending layout id; vertices and
                                             // triangles hold the byte and triangle offsets
    uint64_t items = 0, hash = 0, vbytes = 0, tris = 0; // totals
};
// counts[(segment * n_layouts + layout) * 3]: items, vertices, triangles.  A segment's hash tables hold the smallest power of
// two >= max(64, 2 * its items) entries each (none for an empty segment).  Refused when the totals pass the u32 offsets the
// kernels use.
template <class Fail>
int32_t place_dyn_segments(const uint32_t *counts, uint32_t n_seg, uint32_t n_layouts, const std::vector<fyx_dynamic_layout> &layouts,
                           DynPlacement &p, Fail fail)
{
    const size_t L = n_layouts;
    p = DynPlacement{};
    p.item0.assign(n_seg + 1, 0u);
    p.stream0.assign(n_seg + 1, 0u);
    p.hash0.assign(n_seg, 0u);
    p.hmask.assign(n_seg, 0u);
    p.stream_tri.assign(n_seg * L, 0u);
    p.stream_vtx.assign(n_seg * L, 0u);
    for (uint32_t g = 0; g < n_seg; ++g) {
        p.item0[g] = (uint32_t)p.items;
        p.stream0[g] = (uint32_t)p.streams.size();
        uint64_t ni = 0;
        for (size_t l = 0; l < L; ++l) {
            const uint32_t *k = counts + (g * L + l) * 3;
            p.stream_tri[g * L + l] = (uint32_t)p.tris;
            p.stream_vtx[g * L + l] = p.vbytes;
            if (!k[0]) continue;
            const fyx_dynamic_stream st{(uint32_t)l, layouts[l].stride, k[1], k[2], reinterpret_cast<const void *>(p.vbytes),
                                        reinterpret_cast<const uint32_t *>(p.tris)};
            p.streams.push_back(st);
            ni += k[0];
            p.vbytes = (p.vbytes + (uint64_t)k[1] * st.stride + 15) & ~uint64_t(15);
            p.tris += k[2];
        }
        uint64_t cap = 64;
        while (cap < 2 * ni) cap <<= 1;
        p.hash0[g] = (uint32_t)p.hash;
        p.hmask[g] = (uint32_t)(cap - 1);
        p.hash += ni ? 2 * cap : 0;
        p.items += ni;
    }
    p.item0[n_seg] = (uint32_t)p.items;
    p.stream0[n_seg] = (uint32_t)p.streams.size();
    if (p.items >= (1ull << 31) || p.hash >= (1ull << 32) || p.tris * 3 >= (1ull << 32))
        return fail(FYX_ERR_INVALID_ARGUMENT, "the dynamic batches of one pack are too large (%llu items)", (unsigned long long)p.items);
    return FYX_OK;
}

} // namespace fyx
