// fyx_skin_plan.hpp — the skinning tables of the skinned surfaces: bone slots, k_skin's tiles, the skinned-mesh fold and the
// per-slot / per-surface tables of the bone-matrix blocks.  Host code only, with no CUDA types, so that the CPU tests build
// it with g++ alone.
#pragma once
#include <stdint.h>

#include <algorithm>
#include <vector>

#include "../../include/fyrox_b200.h"

namespace fyx {

constexpr uint32_t kTileQuads = 2048; // up to 8192 vertices per tile (a 5k-vertex surface is one tile)

// One CTA of k_skin: up to kTileQuads four-vertex groups of one surface
struct SkinTile {
    uint32_t bone_off; // first palette entry of the surface
    uint32_t n_bones;
    uint32_t quad_start; // absolute index of the first 4-vertex group
    uint32_t n_quads;
    // blend shapes of the surface (n_shapes = 0: none)
    uint32_t n_shapes;
    uint32_t bs_off;      // index of (shape 0, block 0) of the surface in units of 192 uint2 (one 1536-byte shape block)
    uint32_t bs_blocks;   // 128-vertex blocks per shape
    uint32_t w_off;       // first weight in bs_w
    uint32_t local_quad0; // the tile's first group relative to the surface's first group
    uint32_t vcoded[3];   // bit s: block quad_start / 32 + s is coded (fyx_vcode.cuh); a tile spans at most 65 blocks
};

// One skinned surface (fyx_add_skinned_surface) and where its data lives
struct SkinSurface {
    uint32_t mesh_node;
    std::vector<uint32_t> bones; // node indices
    uint32_t bone_off;           // first palette entry
    uint32_t n_verts;
    uint64_t vert_off;           // first vertex (multiple of 4)
    // N4 blend shapes
    uint32_t n_shapes = 0, bs_blocks = 0, bs_cap = 0; // shapes, 128-vertex blocks per shape, capacity of the region in shape blocks
    uint64_t bs_off = 0;                               // first shape block of the region
    uint32_t w_off = 0, w_cap = 0;
    uint32_t n_bones() const { return (uint32_t)bones.size(); }
};

struct SurfBones { uint32_t bone_off, n_bones; }; // a surface's palette range (the uint2 of the bone-block kernels)

struct SkinPlan {
    std::vector<uint32_t> bone_slot; // [palette entries] slot of the bone node, FYX_NONE = dead or out of range
    std::vector<SkinTile> tiles;     // vcoded is left 0: k_tile_vcode fills it on the device
    // k_fold_bones: per skinned mesh node (alive, in first-surface order) its slot and the bone slots of all its surfaces in
    // surface order (CSR)
    std::vector<uint32_t> fold_node, fold_begin, fold_bone;
    // bones the reference's DFS visits after their mesh keep their pre-update position: per fold entry an index into
    // late_slot (FYX_NONE = not late), and the slots to snapshot
    std::vector<uint32_t> stale_idx, late_slot;
    std::vector<uint32_t> surf_of_slot; // [max(slots, 1)] the node's first surface with bones, FYX_NONE = none
    std::vector<SurfBones> surf_bones;  // [max(surfaces, 1)]
    uint32_t max_bones = 0;             // of the surfaces with vertices
    bool any_blend_shapes = false;      // some surface with vertices has blend shapes
};

// The pre-order rank of every node in the reference's DFS (fyx_set_dfs_order) when it has one entry per node, else null
inline const uint32_t *valid_dfs_rank(const std::vector<uint32_t> &rank, size_t n_nodes) { return rank.size() == n_nodes && n_nodes ? rank.data() : nullptr; }

// dfs_rank: one entry per node (slot_of_node.size()), or null
inline SkinPlan plan_skin(const std::vector<SkinSurface> &surfaces, const std::vector<uint32_t> &slot_of_node, uint32_t n_slots,
                          const uint32_t *dfs_rank)
{
    SkinPlan p;
    auto slot = [&](uint32_t node) { return node < slot_of_node.size() ? slot_of_node[node] : FYX_NONE; };
    p.bone_slot.resize(surfaces.empty() ? 0 : surfaces.back().bone_off + surfaces.back().n_bones()); // surfaces take entries in order
    p.surf_of_slot.assign(std::max<uint32_t>(n_slots, 1), FYX_NONE);
    p.surf_bones.resize(std::max<size_t>(surfaces.size(), 1));
    std::vector<int64_t> fold_of_node(slot_of_node.size(), -1); // node → its fold entry
    std::vector<uint32_t> fold_mesh;                            // node of each fold entry
    std::vector<std::vector<uint32_t>> fold_bone_nodes;
    for (size_t s = 0; s < surfaces.size(); ++s) {
        const SkinSurface &sf = surfaces[s];
        const uint32_t nb = sf.n_bones();
        for (uint32_t b = 0; b < nb; ++b) p.bone_slot[sf.bone_off + b] = slot(sf.bones[b]);
        if (sf.n_verts) {
            const uint32_t quads = (sf.n_verts + 3) / 4;
            const uint32_t nt = (quads + kTileQuads - 1) / kTileQuads, per = (quads + nt - 1) / nt; // tiles, quads per tile
            for (uint32_t t = 0; t < nt; ++t)
                p.tiles.push_back(SkinTile{sf.bone_off, nb, (uint32_t)(sf.vert_off / 4 + (uint64_t)t * per), std::min(per, quads - t * per),
                                           sf.n_shapes, (uint32_t)sf.bs_off, sf.bs_blocks, sf.w_off, t * per, {0, 0, 0}});
            p.max_bones = std::max(p.max_bones, nb);
            p.any_blend_shapes |= sf.n_shapes != 0;
        }
        p.surf_bones[s] = SurfBones{sf.bone_off, nb};
        const uint32_t mesh_slot = slot(sf.mesh_node);
        if (!nb || mesh_slot == FYX_NONE) continue;
        if (p.surf_of_slot[mesh_slot] == FYX_NONE) p.surf_of_slot[mesh_slot] = (uint32_t)s;
        int64_t &fi = fold_of_node[sf.mesh_node];
        if (fi < 0) {
            fi = (int64_t)fold_mesh.size();
            fold_mesh.push_back(sf.mesh_node);
            fold_bone_nodes.emplace_back();
        }
        fold_bone_nodes[fi].insert(fold_bone_nodes[fi].end(), sf.bones.begin(), sf.bones.end());
    }
    p.fold_begin.push_back(0);
    for (size_t m = 0; m < fold_mesh.size(); ++m) {
        p.fold_node.push_back(slot_of_node[fold_mesh[m]]);
        for (uint32_t bn : fold_bone_nodes[m]) {
            const uint32_t bs = slot(bn);
            const bool late = dfs_rank && bs != FYX_NONE && dfs_rank[bn] > dfs_rank[fold_mesh[m]];
            p.stale_idx.push_back(late ? (uint32_t)p.late_slot.size() : FYX_NONE);
            if (late) p.late_slot.push_back(bs);
            p.fold_bone.push_back(bs);
        }
        p.fold_begin.push_back((uint32_t)p.fold_bone.size());
    }
    return p;
}

} // namespace fyx
