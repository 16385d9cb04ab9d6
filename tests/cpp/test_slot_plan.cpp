// The slot planner of fyx_set_topology (fyrox_b200/csrc/fyx_slots.hpp) against the layout rules every kernel relies on, on
// random forests (dead nodes, out-of-range parents, orphans, deep chains, cycles) and on the synthetic scenes of scenegen.
// CPU only.  Prints "slot plan ok" when every check held.
#include <stdio.h>
#include <stdlib.h>

#include <algorithm>
#include <random>
#include <tuple>
#include <vector>

#include "../../fyrox_b200/csrc/fyx_slots.hpp"
#include "../../fyrox_b200/csrc/scenegen.h"

using namespace fyx;

static int g_fail = 0;
#define CHECK(cond, ...)                                                                            \
    do {                                                                                            \
        if (!(cond)) {                                                                              \
            if (g_fail++ < 20) {                                                                    \
                fprintf(stderr, "%s:%d: %s: ", __FILE__, __LINE__, #cond);                          \
                fprintf(stderr, __VA_ARGS__);                                                       \
                fprintf(stderr, "\n");                                                              \
            }                                                                                       \
        }                                                                                           \
    } while (0)

struct Forest {
    std::vector<uint32_t> parent, flags;
    uint32_t capacity() const { return (uint32_t)parent.size(); }
    bool alive(uint32_t i) const { return i < parent.size() && (flags[i] & FYX_NODE_ALIVE); }
};

// depth by walking each chain on its own; -1 = dead, -2 = on or under a cycle
static std::vector<int64_t> naive_depth(const Forest &f)
{
    const uint32_t n = f.capacity();
    std::vector<int64_t> d(n, -1);
    for (uint32_t i = 0; i < n; ++i) {
        if (!f.alive(i)) continue;
        int64_t k = 0;
        uint32_t x = i;
        while (f.parent[x] != FYX_NONE && f.alive(f.parent[x]) && k <= n) {
            x = f.parent[x];
            ++k;
        }
        d[i] = k > n ? -2 : k;
    }
    return d;
}

// The expected layout: levels by depth, each sorted by (parent slot, node index)
static bool check_layout(const Forest &f, const SlotPlan &p, const char *what)
{
    const std::vector<int64_t> depth = naive_depth(f);
    const bool cyclic = std::count(depth.begin(), depth.end(), -2) > 0;
    if (cyclic) {
        CHECK(p.cycle_node != FYX_NONE, "%s: a cycle was not refused", what);
        if (p.cycle_node != FYX_NONE) CHECK(depth[p.cycle_node] == -2, "%s: node %u is not on a cycle", what, p.cycle_node);
        return false;
    }
    CHECK(p.cycle_node == FYX_NONE, "%s: no cycle, but node %u was named", what, p.cycle_node);
    const uint32_t n = f.capacity();
    int64_t max_depth = -1;
    for (int64_t d : depth) max_depth = std::max(max_depth, d);
    std::vector<uint32_t> want_slot(n, FYX_NONE), want_node, want_off(1, 0);
    for (int64_t d = 0; d <= max_depth; ++d) {
        std::vector<std::tuple<uint32_t, uint32_t>> lv; // (parent slot, node)
        for (uint32_t i = 0; i < n; ++i)
            if (depth[i] == d) lv.emplace_back(d ? want_slot[f.parent[i]] : 0u, i);
        std::sort(lv.begin(), lv.end());
        for (auto &e : lv) {
            want_slot[std::get<1>(e)] = (uint32_t)want_node.size();
            want_node.push_back(std::get<1>(e));
        }
        want_off.push_back((uint32_t)want_node.size());
    }
    if (n && max_depth < 0) want_off.push_back(0); // no alive node: one empty level
    CHECK(p.slot_of_node == want_slot, "%s: slot_of_node differs from the (depth, parent slot, node) order", what);
    CHECK(p.node_of_slot == want_node, "%s: node_of_slot differs", what);
    CHECK(p.level_off == want_off, "%s: level_off differs (%zu vs %zu levels)", what, p.level_off.size(), want_off.size());
    CHECK(p.parent.size() == want_node.size(), "%s: parent column size", what);
    // every slot's parent sits in the level before its own
    for (size_t l = 0; l + 1 < p.level_off.size(); ++l)
        for (uint32_t s = p.level_off[l]; s < p.level_off[l + 1] && s < p.parent.size(); ++s) {
            const uint32_t pa = f.parent[p.node_of_slot[s]];
            const uint32_t want = (pa != FYX_NONE && f.alive(pa)) ? p.slot_of_node[pa] : FYX_NONE;
            CHECK(p.parent[s] == want, "%s: parent slot of slot %u", what, s);
            if (l == 0) CHECK(p.parent[s] == FYX_NONE, "%s: slot %u of level 0 has a parent", what, s);
            else CHECK(p.parent[s] >= p.level_off[l - 1] && p.parent[s] < p.level_off[l], "%s: slot %u's parent is not in the level before", what, s);
        }
    return true;
}

// The sub-forest plan's groups, and the rule that picks its first level
static void check_subforest(const SlotPlan &p, int mode, const char *what)
{
    const SubforestLayout sf = plan_subforest(p, mode);
    const uint32_t n_slots = p.n_slots();
    const size_t nlev = p.level_off.size() - 1;
    // the rule, restated: the first level l in [1, nlev - 3] whose sub-trees all have <= kSfCap nodes and with at least 8 deep
    // nodes per node of the level; with mode -1 also no level from l on wider than 131 072
    std::vector<uint32_t> size(n_slots, 1u);
    for (uint32_t s = n_slots; s-- > 0;)
        if (p.parent[s] != FYX_NONE) size[p.parent[s]] += size[s];
    size_t want = 0;
    if (mode != 0 && nlev >= 4)
        for (size_t l = 1; l + 3 <= nlev && !want; ++l) {
            const uint32_t lo = p.level_off[l], hi = p.level_off[l + 1];
            uint32_t widest = 0, mx = 0;
            for (size_t m = l; m < nlev; ++m) widest = std::max(widest, p.level_off[m + 1] - p.level_off[m]);
            for (uint32_t s = lo; s < hi; ++s) mx = std::max(mx, size[s]);
            if (hi > lo && mx <= kSfCap && (uint64_t)(n_slots - lo) >= 8ull * (hi - lo) && (mode == 1 || widest <= 131072u)) want = l;
        }
    CHECK(sf.first_level == want && (sf.n_levels != 0) == (want != 0), "%s, mode %d: first level %u, want %zu", what, mode, sf.first_level,
          want);
    if (!sf.n_levels) {
        CHECK(sf.rng.empty(), "%s, mode %d: ranges without levels", what, mode);
        return;
    }
    CHECK(sf.first_level + sf.n_levels == nlev, "%s, mode %d: the plan does not reach the last level", what, mode);
    const uint32_t G = sf.n_ctas(), L = sf.n_levels;
    CHECK(G >= 1 && sf.rng.size() == (size_t)G * L, "%s, mode %d: %zu ranges for %u groups", what, mode, sf.rng.size(), G);
    // per level, the groups are consecutive ranges covering the level exactly once, each of <= kSfCap nodes
    std::vector<uint32_t> group_of(n_slots, FYX_NONE);
    for (uint32_t l = 0; l < L; ++l) {
        uint32_t at = p.level_off[sf.first_level + l];
        for (uint32_t g = 0; g < G; ++g) {
            const SfRange r = sf.rng[(size_t)g * L + l];
            CHECK(r.begin == at && r.end >= r.begin, "%s, mode %d: group %u level %u starts at %u, not %u", what, mode, g, l, r.begin, at);
            CHECK(r.end - r.begin <= kSfCap, "%s, mode %d: group %u level %u holds %u nodes", what, mode, g, l, r.end - r.begin);
            for (uint32_t s = r.begin; s < r.end && s < n_slots; ++s) group_of[s] = g;
            at = r.end;
        }
        CHECK(at == p.level_off[sf.first_level + l + 1], "%s, mode %d: level %u is not covered", what, mode, l);
    }
    // a sub-tree stays in one group
    for (uint32_t s = p.level_off[sf.first_level + 1]; s < n_slots; ++s)
        CHECK(group_of[s] == group_of[p.parent[s]], "%s, mode %d: slot %u is in group %u, its parent in %u", what, mode, s, group_of[s],
              group_of[p.parent[s]]);
}

static void check(const Forest &f, const char *what)
{
    const SlotPlan p = plan_slots(f.capacity(), f.parent.data(), f.flags.data());
    if (!check_layout(f, p, what)) return;
    for (int mode : {-1, 0, 1}) check_subforest(p, mode, what);
    // the plan is a pure function of its input
    const SlotPlan q = plan_slots(f.capacity(), f.parent.data(), f.flags.data());
    CHECK(q.slot_of_node == p.slot_of_node && q.parent == p.parent, "%s: not stable", what);
}

// a random forest: each node's parent is an earlier node (or none), then some nodes die, some parents point past the end
static Forest random_forest(std::mt19937_64 &rng, uint32_t n, double p_root, double p_dead, double p_bad, uint32_t chain)
{
    Forest f;
    f.parent.resize(n);
    f.flags.assign(n, FYX_NODE_ALIVE);
    std::uniform_real_distribution<double> u(0, 1);
    for (uint32_t i = 0; i < n; ++i) {
        if (i == 0 || u(rng) < p_root) f.parent[i] = FYX_NONE;
        else if (chain && u(rng) < 0.5) f.parent[i] = i - 1 - (uint32_t)(rng() % std::min<uint32_t>(i, chain)); // a deep chain
        else f.parent[i] = (uint32_t)(rng() % i);
        if (u(rng) < p_dead) f.flags[i] = 0;
        if (u(rng) < p_bad) f.parent[i] = n + (uint32_t)(rng() % 5); // out of range
    }
    // shuffle the node indices so that a parent may come after its child
    std::vector<uint32_t> perm(n);
    for (uint32_t i = 0; i < n; ++i) perm[i] = i;
    std::shuffle(perm.begin(), perm.end(), rng);
    Forest g;
    g.parent.resize(n);
    g.flags.resize(n);
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t pa = f.parent[i];
        g.parent[perm[i]] = pa < n ? perm[pa] : pa;
        g.flags[perm[i]] = f.flags[i];
    }
    return g;
}

// the topology of a scenegen scene (a whole one: rank 0 of 1)
static Forest scenegen_forest(uint32_t n_nodes, uint32_t n_units, uint32_t bones)
{
    sg_config cfg{0xF1A0C5, n_nodes, n_units, bones, 4, 0, 1};
    sg_scene *s = sg_create(&cfg);
    Forest f;
    CHECK(s, "scenegen refused %u nodes, %u units of %u bones", n_nodes, n_units, bones);
    if (!s) return f;
    const uint32_t cap = sg_capacity(s);
    f.parent.assign(sg_parent(s), sg_parent(s) + cap);
    f.flags.assign(sg_flags(s), sg_flags(s) + cap);
    sg_free(s);
    return f;
}

int main()
{
    std::mt19937_64 rng(20260917);
    char what[128];
    // shapes
    check(Forest{}, "empty");
    check(Forest{{FYX_NONE}, {0u}}, "one dead node");
    check(Forest{{FYX_NONE, 0, 0}, {FYX_NODE_ALIVE, 0, FYX_NODE_ALIVE}}, "a dead sibling");
    {
        Forest f; // a chain 600 deep under a star
        f.parent.push_back(FYX_NONE);
        for (uint32_t i = 1; i < 400; ++i) f.parent.push_back(0);
        for (uint32_t i = 0; i < 600; ++i) f.parent.push_back(i ? 399 + i : 0);
        f.flags.assign(f.parent.size(), FYX_NODE_ALIVE);
        check(f, "deep chain");
    }
    for (int t = 0; t < 300; ++t) {
        const uint32_t n = 1 + (uint32_t)(rng() % (t < 200 ? 300 : 20000));
        const double p_root = (rng() % 4) * 0.02, p_dead = (rng() % 4) * 0.1, p_bad = (rng() % 3) * 0.02;
        Forest f = random_forest(rng, n, p_root, p_dead, p_bad, (n <= 3000 && rng() % 2) ? 3 : 0); // chains: quadratic checks
        snprintf(what, sizeof what, "random forest %d (%u nodes)", t, n);
        check(f, what);
        if (n >= 3 && t % 3 == 0) { // close a cycle among alive nodes: a node's parent becomes one of its descendants
            uint32_t leaf = (uint32_t)(rng() % n), top = leaf;
            f.flags[leaf] = FYX_NODE_ALIVE;
            for (int k = 0; k < 5 && f.parent[top] < n && f.alive(f.parent[top]); ++k) top = f.parent[top];
            f.parent[top] = leaf;
            snprintf(what, sizeof what, "random forest %d with a cycle", t);
            const SlotPlan p = plan_slots(f.capacity(), f.parent.data(), f.flags.data());
            CHECK(p.cycle_node != FYX_NONE, "%s: not refused", what);
            check(f, what);
        }
    }
    {
        Forest f{{1, 2, 0, 2}, {FYX_NODE_ALIVE, FYX_NODE_ALIVE, 0, FYX_NODE_ALIVE}}; // a "cycle" through a dead node is none
        check(f, "cycle through a dead node");
        CHECK(plan_slots(4, f.parent.data(), f.flags.data()).cycle_node == FYX_NONE, "a dead node closes no cycle");
    }
    // groups of skeletons under wide levels: the deep levels of scenegen's scenes, small enough to run here
    const uint32_t sg[][3] = {{100000, 0, 64}, {100000, 1000, 64}, {200000, 3000, 64}, {200000, 500, 255}, {30000, 200, 7}};
    for (auto &c : sg) {
        snprintf(what, sizeof what, "scenegen %u nodes, %u units of %u bones", c[0], c[1], c[2]);
        check(scenegen_forest(c[0], c[1], c[2]), what);
    }
    // the plan is taken where the rule allows it
    {
        const Forest f = scenegen_forest(100000, 1000, 64);
        const SlotPlan p = plan_slots(f.capacity(), f.parent.data(), f.flags.data());
        CHECK(plan_subforest(p, -1).n_ctas() > 0 && plan_subforest(p, 0).n_ctas() == 0, "scenegen with skeletons: no sub-forest plan");
    }
    if (g_fail) {
        fprintf(stderr, "%d checks failed\n", g_fail);
        return 1;
    }
    printf("slot plan ok\n");
    return 0;
}
