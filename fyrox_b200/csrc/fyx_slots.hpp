// fyx_slots.hpp — the slot layout of a hierarchy (fyx_set_topology) and the sub-forest plan of k_update_subforest.  Host
// code only, with no CUDA types, so that the CPU tests build it with g++ alone.
//
// The layout every kernel relies on: alive nodes get slots sorted by (depth, parent slot, node index), so each hierarchy
// level is one contiguous slot range, a parent always sits in an earlier level and siblings are contiguous.
#pragma once
#include <stdint.h>

#include <algorithm>
#include <vector>

#include "../../include/fyrox_b200.h"

namespace fyx {

constexpr uint32_t kSfCap = 384; // nodes per level and CTA of k_update_subforest (the previous level's matrices stay in shared memory)

struct SlotPlan {
    std::vector<uint32_t> slot_of_node; // [capacity] FYX_NONE = not alive
    std::vector<uint32_t> node_of_slot; // [slots]
    std::vector<uint32_t> level_off;    // [levels + 1] first slot of each depth, then the number of slots
    std::vector<uint32_t> parent;       // [slots] the parent's slot, FYX_NONE = none
    uint32_t cycle_node = FYX_NONE;     // else parent[] has a cycle through this node and the rest of the plan is empty
    uint32_t n_slots() const { return (uint32_t)node_of_slot.size(); }
};

// A node is alive when its FYX_NODE_ALIVE bit is set (flags NULL = every node); a dead or out-of-range parent counts as no
// parent, like Pool::try_borrow failing in graph/mod.rs:1210.
inline SlotPlan plan_slots(uint32_t capacity, const uint32_t *parent, const uint32_t *flags)
{
    auto alive = [&](uint32_t i) { return i < capacity && (!flags || (flags[i] & FYX_NODE_ALIVE)); };
    SlotPlan p;
    // depth of every alive node, along its parent chain
    std::vector<int32_t> depth(capacity, -1);
    std::vector<uint32_t> path;
    uint32_t max_depth = 0;
    for (uint32_t i = 0; i < capacity; ++i) {
        if (!alive(i) || depth[i] >= 0) continue;
        path.clear();
        uint32_t n = i;
        int32_t base = -1;
        while (true) {
            if (depth[n] >= 0) { base = depth[n]; break; }
            if (depth[n] == -2) {
                p.cycle_node = n;
                return p;
            }
            depth[n] = -2;
            path.push_back(n);
            const uint32_t pa = parent[n];
            if (pa == FYX_NONE || !alive(pa)) break;
            n = pa;
        }
        for (size_t k = path.size(); k-- > 0;) {
            base += 1;
            depth[path[k]] = base;
            max_depth = std::max<uint32_t>(max_depth, (uint32_t)base);
        }
    }
    // counting sort by depth, stable in node index
    std::vector<uint32_t> &level_off = p.level_off, &slot_of_node = p.slot_of_node, &node_of_slot = p.node_of_slot;
    level_off.assign(capacity ? max_depth + 2 : 1, 0);
    uint32_t n_slots = 0;
    for (uint32_t i = 0; i < capacity; ++i)
        if (alive(i)) { level_off[depth[i] + 1]++; n_slots++; }
    for (size_t l = 1; l < level_off.size(); ++l) level_off[l] += level_off[l - 1];
    std::vector<uint32_t> cursor(level_off.begin(), level_off.end());
    slot_of_node.assign(capacity, FYX_NONE);
    node_of_slot.resize(n_slots);
    for (uint32_t i = 0; i < capacity; ++i)
        if (alive(i)) {
            const uint32_t s = cursor[depth[i]]++;
            slot_of_node[i] = s;
            node_of_slot[s] = i;
        }
    // within a level, order by parent slot (counting sort, stable in node index): siblings become contiguous, so a warp's
    // gather of parent rows touches one or two parents instead of 32
    std::vector<uint32_t> tmp, cnt;
    for (size_t d = 1; d + 1 < level_off.size(); ++d) {
        const uint32_t plo = level_off[d - 1], phi = level_off[d], lo = level_off[d], hi = level_off[d + 1];
        if (hi - lo < 2) continue;
        cnt.assign((size_t)(phi - plo) + 1, 0);
        for (uint32_t s = lo; s < hi; ++s) cnt[slot_of_node[parent[node_of_slot[s]]] - plo + 1]++;
        for (size_t k = 1; k < cnt.size(); ++k) cnt[k] += cnt[k - 1];
        tmp.resize(hi - lo);
        for (uint32_t s = lo; s < hi; ++s) {
            const uint32_t i = node_of_slot[s];
            tmp[cnt[slot_of_node[parent[i]] - plo]++] = i;
        }
        for (uint32_t k = 0; k < hi - lo; ++k) {
            node_of_slot[lo + k] = tmp[k];
            slot_of_node[tmp[k]] = lo + k;
        }
    }
    p.parent.resize(n_slots);
    for (uint32_t s = 0; s < n_slots; ++s) {
        const uint32_t pa = parent[node_of_slot[s]];
        p.parent[s] = (pa != FYX_NONE && alive(pa)) ? slot_of_node[pa] : FYX_NONE;
    }
    return p;
}

// One record per node index, for what the setters keep on the host by node: light sources, CSM options, cameras, reflection
// probes, node surfaces, pruner marks, quad nodes.  `def` is the record of a node that was never given one.  Across
// fyx_set_topology a record stays with its node index while the node is alive before and after the call; every other index
// starts again from `def`, as in the slot columns.
template <class T> struct NodeRecords {
    T def;
    std::vector<T> rec; // by node index; the indices past its end hold `def`
    explicit NodeRecords(const T &v) : def(v) {}
    const T &operator[](uint32_t node) const { return node < rec.size() ? rec[node] : def; }
    void set(uint32_t node, const T &v)
    {
        if (node >= rec.size()) rec.resize(node + 1, def);
        rec[node] = v;
    }
    int32_t check(fyx_ctx *c, uint32_t count, const uint32_t *idx) const; // every node listed (idx NULL = 0..count-1) is in range
    // keep(record) trims a record that stays to what it keeps.  Only the records that restart are written.
    template <class Keep> void topology_changed(const std::vector<uint32_t> &old_slot_of_node, const std::vector<uint32_t> &new_slot_of_node, Keep keep)
    {
        if (rec.size() > new_slot_of_node.size()) rec.resize(new_slot_of_node.size());
        for (size_t i = 0; i < rec.size(); ++i) {
            if (i < old_slot_of_node.size() && old_slot_of_node[i] != FYX_NONE && new_slot_of_node[i] != FYX_NONE) keep(rec[i]);
            else rec[i] = def;
        }
    }
    void topology_changed(const std::vector<uint32_t> &old_slot_of_node, const std::vector<uint32_t> &new_slot_of_node)
    {
        topology_changed(old_slot_of_node, new_slot_of_node, [](T &) {});
    }
    // f(node, slot, record) for the record of every alive node, in pool order
    template <class F> void for_alive(const std::vector<uint32_t> &slot_of_node, F f)
    {
        const size_t n = std::min(rec.size(), slot_of_node.size());
        for (size_t node = 0; node < n; ++node)
            if (slot_of_node[node] != FYX_NONE) f((uint32_t)node, slot_of_node[node], rec[node]);
    }
};

struct SfRange {
    uint32_t begin, end; // slots [begin, end) of one level of one group
};
struct SubforestLayout {
    uint32_t first_level = 0, n_levels = 0; // deep levels = [first_level, first_level + n_levels); n_levels 0 = no plan
    std::vector<SfRange> rng;               // [group][level]: one group per CTA
    uint32_t n_ctas() const { return n_levels ? (uint32_t)(rng.size() / n_levels) : 0u; }
};

// From the first level on whose sub-trees are all small (<= kSfCap nodes) and numerous relative to the level's width
// (skeletons under a wide level of meshes), whole sub-trees are grouped so that no level of a group has more than kSfCap
// nodes; a group is one CTA of k_update_subforest.  Slots are sorted by (depth, parent slot), so the nodes of a group form
// one contiguous slot range in every level.  mode -1: only where every deep level is narrow (<= 131 072 nodes: a wide
// level keeps a launch of its own busy, only narrow ones are launch-bound); 1: wherever such a level exists; 0: never.
inline SubforestLayout plan_subforest(const SlotPlan &p, int mode)
{
    SubforestLayout sf;
    const std::vector<uint32_t> &level_off = p.level_off;
    const uint32_t n_slots = p.n_slots();
    const size_t nlev = level_off.size() ? level_off.size() - 1 : 0;
    if (mode == 0 || nlev < 4 || !n_slots) return sf;
    std::vector<uint32_t> size(n_slots, 1u);
    for (uint32_t s = n_slots; s-- > 0;)
        if (p.parent[s] != FYX_NONE) size[p.parent[s]] += size[s];
    // widest level at or below l
    std::vector<uint32_t> widest(nlev + 1, 0u);
    for (size_t l = nlev; l-- > 0;) widest[l] = std::max(widest[l + 1], level_off[l + 1] - level_off[l]);
    size_t pick = 0;
    for (size_t l = 1; l + 3 <= nlev; ++l) {
        uint32_t mx = 0;
        for (uint32_t s = level_off[l]; s < level_off[l + 1]; ++s) mx = std::max(mx, size[s]);
        const uint64_t cnt = level_off[l + 1] - level_off[l], deep = n_slots - level_off[l];
        if (cnt && mx <= kSfCap && deep >= 8 * cnt && (mode == 1 || widest[l] <= 131072u)) { pick = l; break; }
    }
    if (!pick) return sf;
    const uint32_t levels = (uint32_t)(nlev - pick), base = level_off[pick];
    sf.first_level = (uint32_t)pick;
    sf.n_levels = levels;
    // per level, how many nodes each sub-tree of level `pick` has there; the sub-trees in slot order own consecutive ranges
    const uint32_t n_tiles = level_off[pick + 1] - base;
    std::vector<uint32_t> tile_of(n_slots - base);
    std::vector<uint32_t> cnt((size_t)n_tiles * levels, 0u);
    for (uint32_t s = base; s < n_slots; ++s) {
        const uint32_t rel = s - base;
        tile_of[rel] = (s < level_off[pick + 1]) ? rel : tile_of[p.parent[s] - base];
    }
    for (size_t l = pick; l < nlev; ++l)
        for (uint32_t s = level_off[l]; s < level_off[l + 1]; ++s) cnt[(size_t)tile_of[s - base] * levels + (l - pick)]++;
    std::vector<uint32_t> cursor(levels), acc(levels, 0u);
    for (uint32_t li = 0; li < levels; ++li) cursor[li] = level_off[pick + li];
    auto close_group = [&]() {
        for (uint32_t li = 0; li < levels; ++li) {
            sf.rng.push_back(SfRange{cursor[li], cursor[li] + acc[li]});
            cursor[li] += acc[li];
            acc[li] = 0;
        }
    };
    for (uint32_t t = 0; t < n_tiles; ++t) {
        bool fits = true;
        for (uint32_t li = 0; li < levels; ++li)
            if (acc[li] + cnt[(size_t)t * levels + li] > kSfCap) fits = false;
        if (!fits) close_group();
        for (uint32_t li = 0; li < levels; ++li) acc[li] += cnt[(size_t)t * levels + li];
    }
    close_group();
    return sf;
}

} // namespace fyx
